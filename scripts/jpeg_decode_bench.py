"""JPEG decode throughput and latency: image_io.decode_jpegs (one batched call) and decode_jpeg (one file), next to
cv2.imread on 1 and N host threads. One process, one GPU.

  OUT=jpeg_bench.json python scripts/jpeg_decode_bench.py                 # ITERS=10 ROUNDS=3
  python scripts/jpeg_decode_bench.py --single-only                        # only the decode_jpeg arm (any checkout)

Input: 64 synthetic 540 x 720 RGB frames (seeded band-limited texture + per-pixel noise), JPEG quality 95, 4:2:0,
held as bytes in host memory. decode_jpegs at batches of 1, 16 and 64, gray and RGB; decode_jpeg per file, gray.
Each timed window is ITERS calls after a warm-up, between CUDA events on the current stream (the decoded images stay
on the device); the median over ROUNDS windows is reported. The card's name and power limit are read in the same run.
Prints one JSON document (and writes it to OUT if set)."""
import json
import os
import subprocess
import sys
import time
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


def frames():
    rng = np.random.default_rng(0)
    out = []
    for _ in range(N):
        im = synth.make_texture(rng, H, W).astype(np.int32) + rng.integers(-12, 12, (H, W, 3))
        ok, buf = cv2.imencode(".jpg", im.clip(0, 255).astype(np.uint8),
                               [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
        assert ok
        out.append(buf.tobytes())
    return out


def ms_per_call(fn):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(ITERS):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / ITERS)
    return float(np.median(res))


def host_ms(fn):
    fn()
    res = []
    for _ in range(ROUNDS):
        t0 = time.perf_counter()
        for _ in range(max(1, ITERS // 5)):
            fn()
        res.append((time.perf_counter() - t0) * 1e3 / max(1, ITERS // 5))
    return float(np.median(res))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unavailable ({e})"
    return q


def main():
    assert torch.cuda.is_available(), "jpeg_decode_bench needs a CUDA device"
    data = frames()
    res = {"card": card(), "frames": f"{N} x {W}x{H} q95 4:2:0", "mean_bytes": float(np.mean([len(d) for d in data]))}
    res["decode_jpeg_ms_per_image"] = ms_per_call(lambda: [image_io.decode_jpeg(d) for d in data[:8]]) / 8
    if "--single-only" not in sys.argv:
        for rgb in (False, True):
            for b in (1, 16, 64):
                ms = ms_per_call(lambda: image_io.decode_jpegs(data[:b], rgb=rgb))
                res[f"decode_jpegs_{'rgb' if rgb else 'gray'}_b{b}"] = {"ms_per_batch": ms, "images_per_s": b / ms * 1e3}
        buf = [np.frombuffer(d, np.uint8) for d in data]
        res["cv2_1thread_ms_per_image"] = host_ms(lambda: [cv2.imdecode(b, cv2.IMREAD_GRAYSCALE) for b in buf[:16]]) / 16
        nt = os.cpu_count() or 1
        with ThreadPoolExecutor(nt) as ex:
            ms = host_ms(lambda: list(ex.map(lambda b: cv2.imdecode(b, cv2.IMREAD_GRAYSCALE), buf)))
        res[f"cv2_{nt}threads_images_per_s"] = N / ms * 1e3
    s = json.dumps(res, indent=1)
    print(s)
    if os.environ.get("OUT"):
        with open(os.environ["OUT"], "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
