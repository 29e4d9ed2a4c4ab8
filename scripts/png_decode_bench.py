"""Depth-PNG decode throughput: image_io.decode_pngs (one batched GPU call) next to cv2.imdecode(IMREAD_UNCHANGED) on 1
and 8 host threads, in one process on one GPU.

  OUT=png_bench.json python scripts/png_decode_bench.py             # ITERS=10 ROUNDS=3

Input: 64 Map-free-sized 720 x 540 16-bit depth maps (synth.make_depth in millimetres, zeros included), encoded two
ways, since the dataset's encoder is not known: cv2.imencode's defaults (Sub filter on every row, zlib level 1, Z_RLE)
and zlib level 6 with libpng's per-row adaptive filter choice (the filter with the least sum of |signed byte|). The GPU
rate is images/s at batches of 1, 16 and 64, timed with the host clock around the call plus a device synchronise, so
host parsing and staging count; every file must decode on the GPU (a host fallback would be timed as GPU work). The
per-kernel times (CRC, inflate, unfilter) are CUDA events around each kernel of batch-64 calls
(mfr_debug_png_kernel_ms). The card's name and power limit are read in the same run. Prints one JSON document (and writes it to OUT)."""
import json
import os
import struct
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mfr_b200  # noqa: E402,F401
from mfr_b200 import image_io, synth  # noqa: E402

ITERS = int(os.environ.get("ITERS", 10))
ROUNDS = int(os.environ.get("ROUNDS", 3))
N, H, W = 64, 720, 540


def _chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def adaptive_png(mm):
    """16-bit gray PNG with libpng's adaptive row filters and zlib level 6."""
    raw = mm.astype(">u2").view(np.uint8).reshape(mm.shape[0], -1).astype(np.int32)
    rows = []
    for r in range(raw.shape[0]):
        cur = raw[r]
        up = raw[r - 1] if r else np.zeros_like(cur)
        left = np.concatenate([[0, 0], cur[:-2]])
        ul = np.concatenate([[0, 0], up[:-2]])
        p = left + up - ul
        pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
        paeth = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
        cands = [cur, cur - left, cur - up, cur - (left + up) // 2, cur - paeth]
        cands = [(c & 255).astype(np.uint8) for c in cands]
        cost = [np.abs(c.astype(np.int8).astype(np.int32)).sum() for c in cands]
        f = int(np.argmin(cost))
        rows.append(bytes([f]) + cands[f].tobytes())
    z = zlib.compress(b"".join(rows), 6)
    h, w = mm.shape
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 16, 0, 0, 0, 0)) + _chunk(b"IDAT", z) +
            _chunk(b"IEND", b""))


def frames():
    rng = np.random.default_rng(0)
    mms = [np.round(synth.make_depth(rng, H, W).astype(np.float64) * 1000).astype(np.uint16) for _ in range(N)]
    return {"cv2_default": [cv2.imencode(".png", m)[1].tobytes() for m in mms],
            "zlib6_adaptive": [adaptive_png(m) for m in mms]}


def wall_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(ROUNDS):
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        res.append((time.perf_counter() - t0) * 1e3 / iters)
    return float(np.median(res))


def host_ms(fn):
    fn()
    res = []
    for _ in range(ROUNDS):
        t0 = time.perf_counter()
        fn()
        res.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(res))


def kernel_ms(data):
    """Median over ITERS batch-64 calls of each decoder kernel's time (CUDA events around each kernel)."""
    import ctypes
    from mfr_b200 import lib
    dev = torch.device("cuda", torch.cuda.current_device())
    ms = (ctypes.c_float * 3)()
    res = []
    for _ in range(ITERS):
        image_io.decode_pngs(data)
        dec = image_io._decoder("png", dev, len(data), 1, 1)
        lib.check(lib.load().mfr_debug_png_kernel_ms(dec.h, ms), "mfr_debug_png_kernel_ms")
        res.append(list(ms))
    med = np.median(np.array(res), 0)
    return {"crc": float(med[0]), "inflate": float(med[1]), "unfilter": float(med[2])}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    assert torch.cuda.is_available(), "png_decode_bench needs a CUDA device"
    res = {"card": card(), "frames": f"{N} x {W}x{H} 16-bit depth PNG"}
    for enc, data in frames().items():
        r = res[enc] = {"mean_bytes": float(np.mean([len(d) for d in data]))}
        got = image_io.decode_pngs(data)
        ref = [cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_UNCHANGED) for d in data]
        assert all(np.array_equal(g.cpu().numpy(), x) for g, x in zip(got, ref))
        # no file may fall back to the host: the device status of every frame
        dev = torch.device("cuda", torch.cuda.current_device())
        _, status = image_io._png_batch(data, 0, dev, lambda i, w, h, d: torch.empty((h, w), dtype=torch.uint16, device=dev))
        assert not any(status), f"device rejected frames: {status}"
        for b in (1, 16, 64):
            ms = wall_ms(lambda: image_io.decode_pngs(data[:b]), max(3, ITERS * 4 // b))
            r[f"gpu_b{b}"] = {"ms_per_batch": ms, "images_per_s": b / ms * 1e3}
        r["kernel_ms_b64"] = kernel_ms(data)
        buf = [np.frombuffer(d, np.uint8) for d in data]
        r["cv2_1thread_images_per_s"] = 16 / host_ms(lambda: [cv2.imdecode(x, cv2.IMREAD_UNCHANGED) for x in buf[:16]]) * 1e3
        with ThreadPoolExecutor(8) as ex:
            ms = host_ms(lambda: list(ex.map(lambda x: cv2.imdecode(x, cv2.IMREAD_UNCHANGED), buf)))
        r["cv2_8threads_images_per_s"] = N / ms * 1e3
    s = json.dumps(res, indent=1)
    print(s)
    if os.environ.get("OUT"):
        with open(os.environ["OUT"], "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
