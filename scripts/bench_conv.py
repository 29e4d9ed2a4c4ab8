"""Times the wgmma conv kernel at LoFTR layer shapes (CUDA events) and cuDNN beside it."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import mfr_b200
from mfr_b200 import lib as mfr

lib = mfr.load()
SHAPES = [  # N,H,W,Cin,Cout,R,stride
    (2, 360, 272, 128, 128, 3, 1),
    (2, 360, 272, 128, 196, 3, 2),
    (2, 180, 136, 196, 196, 3, 1),
    (2, 180, 136, 196, 256, 3, 2),
    (2, 90, 68, 256, 256, 3, 1),
    (2, 360, 272, 128, 196, 1, 1),
    (2, 360, 272, 196, 196, 3, 1),
    (2, 360, 272, 196, 128, 3, 1),
    (2, 1, 6120, 256, 256, 1, 1),
    (2, 1, 6120, 512, 512, 1, 1),
]
for (N, H, W, Cin, Cout, R, s) in SHAPES:
    x = torch.randn(N, H, W, Cin, device="cuda")
    w = torch.randn(Cout, R, R, Cin, device="cuda") / (R * R * Cin) ** 0.5
    pad = R // 2
    Ho = (H + 2 * pad - R) // s + 1
    Wo = (W + 2 * pad - R) // s + 1
    out = torch.empty(N, Ho, Wo, Cout, device="cuda")
    def run():
        mfr.check(lib.mfr_conv2d_nhwc_tf32(mfr.ptr(x), N, H, W, Cin, Cin, mfr.ptr(w), Cout, R, R, s, pad, 0,
                                 None, None, Cout, 1, 1.0, mfr.ptr(out), Cout, mfr.cur_stream()))
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    fl = 2.0 * N * Ho * Wo * Cout * Cin * R * R
    # cuDNN channels-last TF32 beside it
    torch.backends.cudnn.allow_tf32 = True
    xc = x.permute(0, 3, 1, 2)  # NCHW view with channels_last strides
    wc = w.permute(0, 3, 1, 2)
    for _ in range(3):
        F.conv2d(xc, wc, None, stride=s, padding=pad)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(10):
        F.conv2d(xc, wc, None, stride=s, padding=pad)
    e1.record(); torch.cuda.synchronize()
    ms2 = e0.elapsed_time(e1) / 10
    print(f"{(N,H,W,Cin,Cout,R,s)}: ours {ms:.3f} ms {fl/ms/1e9:.1f} TF/s | cudnn {ms2:.3f} ms {fl/ms2/1e9:.1f} TF/s", flush=True)
