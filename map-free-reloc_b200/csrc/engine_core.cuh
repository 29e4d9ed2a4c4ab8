// Host-side machinery shared by the LoFTR, SuperPoint + SuperGlue and SIFT engines (no kernels): zeroed device
// buffers with a debug registry, the fp32 weight table and the GEMM copies derived from it, launch lists and the CUDA
// graphs they are replayed through.
#pragma once
#include <cstdint>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "loftr_ops.cuh"   // weights_to_bf16, rows_split3

namespace mfr {

// Device buffers, zeroed when allocated and freed with the arena. Named buffers are listed for the debug ABI with
// their size in 4-byte words, whatever their element type.
struct DeviceArena {
  explicit DeviceArena(int* rc) : rc(rc) {}
  DeviceArena(const DeviceArena&) = delete;
  ~DeviceArena() { for (void* p : ptrs) cudaFree(p); }

  template <class T>
  T* alloc(size_t n, const char* name = nullptr) {
    void* p = nullptr;
    const size_t bytes = n * sizeof(T);
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
      fprintf(stderr, "[mfr_b200] cudaMalloc of %zu bytes failed (%s)\n", bytes, name ? name : "");
      *rc = MFR_ERR_CUDA;
      return nullptr;
    }
    cudaMemset(p, 0, bytes);
    ptrs.push_back(p);
    if (name) named[name] = {static_cast<float*>(p), static_cast<long long>(bytes / 4)};
    return static_cast<T*>(p);
  }
  int debug_tensor(const char* name, float** ptr, long long* numel) const {
    if (!name || !ptr || !numel) return MFR_ERR_ARG;
    auto it = named.find(name);
    if (it == named.end()) return MFR_ERR_ARG;
    *ptr = it->second.first;
    *numel = it->second.second;
    return MFR_OK;
  }

  int* rc;
  std::vector<void*> ptrs;
  std::map<std::string, std::pair<float*, long long>> named;
};

// Named fp32 tensors at 64-float-aligned offsets of one device blob, uploaded one by one through the ABI.
struct WeightTable {
  struct Entry { std::string name; size_t numel, offset; bool set; };
  explicit WeightTable(int* rc) : rc(rc) {}

  void add(const std::string& name, size_t numel) {
    index[name] = entries.size();
    entries.push_back({name, numel, total, false});
    total += (numel + 63) / 64 * 64;
  }
  float* alloc(DeviceArena& mem) { return blob = mem.alloc<float>(total, "weights"); }
  float* operator[](const std::string& name) const {
    auto it = index.find(name);
    if (it == index.end()) {
      fprintf(stderr, "[mfr_b200] unknown weight %s\n", name.c_str());
      *rc = MFR_ERR_ARG;
      return blob;
    }
    return blob + entries[it->second].offset;
  }
  int count() const { return static_cast<int>(entries.size()); }
  const char* name(int i) const { return entries[i].name.c_str(); }
  long long numel(int i) const { return static_cast<long long>(entries[i].numel); }
  // Uploads tensor i from host memory. Every upload starts a new generation: what was derived from the old weights
  // (GEMM copies, an encoded map frame) is stale.
  int set(int i, const float* host, long long n, cudaStream_t st) {
    if (i < 0 || i >= count() || n != numel(i)) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaMemcpyAsync(blob + entries[i].offset, host, n * 4, cudaMemcpyHostToDevice, st));
    MFR_CUDA_CHECK(cudaStreamSynchronize(st));
    entries[i].set = true;
    ++generation;
    return MFR_OK;
  }
  // every tensor has been uploaded at least once
  bool complete() const {
    for (const auto& e : entries)
      if (!e.set) return false;
    return true;
  }

  int* rc;
  std::vector<Entry> entries;
  std::map<std::string, size_t> index;
  float* blob = nullptr;
  size_t total = 0;           // floats
  long long generation = 0;   // uploads so far
};

// Copies of GEMM weights in the layout the tensor-core GEMMs read instead of the fp32 table, one per weight name:
//  - kBf16:   bf16 rows with the row stride padded to a multiple of 8 elements (16-byte TMA strides);
//  - kSplit3: the [hi | hi | lo] 3xTF32 split of every row (3 * cin floats).
// The steps bake the copies' addresses into their TMA descriptors, so the blob is sized from the weight table before
// any step is built, and a registration that does not fit fails the build.
struct DerivedWeights {
  enum Kind { kBf16, kSplit3 };
  struct Entry { std::string name; long long rows; int cin; size_t off; };   // off: elements
  explicit DerivedWeights(int* rc) : rc(rc) {}

  int ld(int cin) const { return kind == kBf16 ? (cin + 7) / 8 * 8 : 3 * cin; }
  size_t esize() const { return kind == kBf16 ? 2 : 4; }
  // A row takes at most 2 (bf16, cin >= 4) or 3 (split) elements per fp32 weight element, plus the 64-element alignment.
  void alloc(DeviceArena& mem, const WeightTable& w, Kind k) {
    kind = k;
    cap = (kind == kBf16 ? 2 : 3) * w.total + 64 * w.entries.size();
    blob = mem.alloc<char>(cap * esize(), kind == kBf16 ? "weights_bf16" : "weights_split3");
  }
  // Row `row` of the copy of weight `name` ([rows][cin] in the table); a second request for a name returns the same copy.
  const float* get(const WeightTable& w, const std::string& name, long long rows, int cin, long long row = 0) {
    size_t off = used;
    bool found = false;
    for (const auto& e : entries)
      if (e.name == name) { off = e.off; found = true; }
    if (!found) {
      const size_t n = (static_cast<size_t>(rows) * ld(cin) + 63) / 64 * 64;
      auto it = w.index.find(name);
      if (used + n > cap || it == w.index.end() || static_cast<size_t>(rows) * cin != w.entries[it->second].numel) {
        fprintf(stderr, "[mfr_b200] no room for the derived copy of %s\n", name.c_str());
        *rc = MFR_ERR_ARG;
        return reinterpret_cast<const float*>(blob);
      }
      entries.push_back({name, rows, cin, off});
      used += n;
    }
    return reinterpret_cast<const float*>(blob + (off + static_cast<size_t>(row) * ld(cin)) * esize());
  }
  // Converts every registered weight again if the table changed since the last call. Runs outside any capture.
  int rebuild(const WeightTable& w, cudaStream_t st) {
    if (built == w.generation) return MFR_OK;
    for (const auto& e : entries) {
      const int r = kind == kBf16
          ? weights_to_bf16(w[e.name], blob + e.off * 2, e.rows, e.cin, ld(e.cin), st)
          : rows_split3(w[e.name], e.cin, 0, reinterpret_cast<float*>(blob) + e.off, e.rows, 1, e.cin, 1, nullptr, st);
      if (r != MFR_OK) return r;
    }
    built = w.generation;
    return MFR_OK;
  }

  int* rc;
  Kind kind = kBf16;
  char* blob = nullptr;
  size_t cap = 0, used = 0;   // elements
  long long built = -1;       // weight generation the copies were made from
  std::vector<Entry> entries;
};

// One step of a launch list, with what the profiles report about it.
struct Step {
  std::function<int(cudaStream_t)> f;
  std::string name;
  int launches = 1;               // kernels the step launches
  int kind = 0;                   // 1 = tensor-core conv / GEMM launch, 0 = SIMT kernel(s)
  double flops = 0;               // algorithmic FLOPs; per live row when dyn_rows is set
  const int* dyn_rows = nullptr;  // device row count (per image) or null
  int dyn_images = 0;
  int group = 0;                  // timed_run measures consecutive steps of one group together
};

struct LaunchList {
  std::vector<Step> steps;

  // appends a step whose group is its index
  Step& push(std::function<int(cudaStream_t)> f, std::string name = "", int launches = 1) {
    Step s;
    s.f = std::move(f); s.name = std::move(name); s.launches = launches; s.group = size();
    steps.push_back(std::move(s));
    return steps.back();
  }
  // appends steps [begin, end) of another list
  void append(const LaunchList& o, size_t begin, size_t end) {
    steps.insert(steps.end(), o.steps.begin() + begin, o.steps.begin() + end);
  }
  int size() const { return static_cast<int>(steps.size()); }
  int launches() const {
    int n = 0;
    for (const auto& s : steps) n += s.launches;
    return n;
  }
  int run(cudaStream_t st, size_t begin = 0, size_t end = SIZE_MAX) const {
    for (size_t i = begin; i < steps.size() && i < end; ++i) {
      const int rc = steps[i].f(st);
      if (rc != MFR_OK) return rc;
    }
    return MFR_OK;
  }
};

// Eager run with a CUDA event wherever a step's group differs from the previous step's. ms[g] = device time of group g
// (groups ascend from 0; a group without steps takes 0).
inline int timed_run(const LaunchList& list, cudaStream_t st, std::vector<float>& ms) {
  const int n = list.steps.empty() ? 0 : list.steps.back().group + 1;
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) MFR_CUDA_CHECK(cudaEventCreate(&e));
  int g = 0, rc = cudaEventRecord(ev[0], st) == cudaSuccess ? MFR_OK : MFR_ERR_CUDA;
  for (const auto& s : list.steps) {
    if (rc != MFR_OK) break;
    while (g < s.group) cudaEventRecord(ev[++g], st);
    rc = s.f(st);
  }
  while (g < n) cudaEventRecord(ev[++g], st);
  if (cudaEventSynchronize(ev[n]) != cudaSuccess && rc == MFR_OK) rc = MFR_ERR_CUDA;
  ms.assign(n, 0.f);
  for (int i = 0; i < n && rc == MFR_OK; ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

// A launch list's CUDA graph, captured on its first launch.
struct GraphExec {
  GraphExec() = default;
  GraphExec(const GraphExec&) = delete;
  ~GraphExec() { if (exec) cudaGraphExecDestroy(exec); }

  // Eager while use_graph is off. The first launch runs the list eagerly (which loads its kernels and sets their
  // attributes outside the capture, and gives this call's results), then captures it. If the capture fails, use_graph
  // is turned off and the list runs eagerly.
  int launch(const LaunchList& list, cudaStream_t st, bool& use_graph, const char* engine) {
    if (!use_graph) return list.run(st);
    if (exec) {
      MFR_CUDA_CHECK(cudaGraphLaunch(exec, st));
      return MFR_OK;
    }
    int rc = list.run(st);
    if (rc != MFR_OK) return rc;
    MFR_CUDA_CHECK(cudaStreamSynchronize(st));
    cudaGraph_t g;
    MFR_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    rc = list.run(st);
    const cudaError_t e = cudaStreamEndCapture(st, &g);
    if (rc != MFR_OK || e != cudaSuccess) {
      fprintf(stderr, "[mfr_b200] %s graph capture failed (%d, %s); running eagerly\n", engine, rc, cudaGetErrorString(e));
      use_graph = false;
      cudaGetLastError();
      return list.run(st);
    }
    MFR_CUDA_CHECK(cudaGraphInstantiate(&exec, g, 0));
    cudaGraphDestroy(g);
    return MFR_OK;
  }

  cudaGraphExec_t exec = nullptr;
};

// What the ABI operations shared by every engine see of it: weight enumeration and upload, debug buffers, the graph
// switch and the forward list's launch counts.
struct EngineCore {
  EngineCore() = default;
  EngineCore(const EngineCore&) = delete;

  int rc = MFR_OK;        // first error met while building the engine
  bool use_graph = true;
  DeviceArena mem{&rc};
  WeightTable weights{&rc};
  LaunchList steps;       // the forward
};

}  // namespace mfr
