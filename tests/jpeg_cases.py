"""JPEG files generated with cv2.imencode for the decoder tests (tests/test_jpeg_host.py, tests/test_jpeg_gpu.py), and
cv2.imread's result for them: the decoder's acceptance bar is byte equality with the installed OpenCV (4.13.0, bundling
libjpeg-turbo 3.1.2)."""
import struct

import cv2
import numpy as np

from helpers import synth

SIZES = [(720, 540), (540, 720), (333, 250), (17, 9), (8, 8), (1, 1), (2, 3)]      # (h, w)
SAMPLING = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}


def content(kind, h, w, seed=0):
    """RGB uint8 [h, w, 3]: band-limited texture, per-pixel noise, or hard black / white edges (IDCT overshoot)."""
    rng = np.random.default_rng(seed + 7 * h + w)
    if kind == "texture":
        return synth.make_texture(rng, h, w)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    im = (((yy // 3) + (xx // 5)) % 2 * 255).astype(np.uint8)
    im[(xx * 7 + yy * 3) % 11 == 0] = 0
    return np.stack([im, 255 - im, im], -1)


def encode(rgb, params=(), gray=False):
    img = cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY) if gray else rgb[:, :, ::-1]
    ok, buf = cv2.imencode(".jpg", img, list(params))
    assert ok
    return buf.tobytes()


def with_orientation(data, orient):
    """``data`` with an APP1 Exif segment (IFD0 with only the Orientation tag) inserted after SOI."""
    tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, orient, 0) \
        + struct.pack("<I", 0)
    payload = b"Exif\x00\x00" + tiff
    return data[:2] + b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload + data[2:]


def with_16bit_dqt(data):
    """``data`` with every 8-bit quantisation table rewritten as a 16-bit one (same values)."""
    out, i = bytearray(data[:2]), 2
    while data[i + 1] != 0xDA:
        n = int.from_bytes(data[i + 2:i + 4], "big")
        seg = data[i:i + 2 + n]
        if data[i + 1] == 0xDB:
            body, o = bytearray(), 4
            while o < len(seg):
                pq, tq = seg[o] >> 4, seg[o] & 15
                vals = seg[o + 1:o + 1 + 64 * (pq + 1)]
                body.append(0x10 | tq)
                body += vals if pq else b"".join(v.to_bytes(2, "big") for v in vals)
                o += 1 + 64 * (pq + 1)
            seg = b"\xff\xdb" + (len(body) + 2).to_bytes(2, "big") + bytes(body)
        out += seg
        i += 2 + n
    return bytes(out + data[i:])


def cv2_decode(data, rgb):
    """What cv2.imread gives for the file: gray [h, w] (IMREAD_GRAYSCALE) or RGB [h, w, 3] (IMREAD_COLOR, BGR -> RGB)."""
    im = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR if rgb else cv2.IMREAD_GRAYSCALE)
    return np.ascontiguousarray(im[:, :, ::-1]) if rgb else im


def matrix():
    """[(name, bytes)] of supported files: every size x sampling x content at quality 95, the quality sweep, separate
    luma / chroma qualities, optimised tables, restart intervals and one-component files."""
    cases = []
    for h, w in SIZES:
        for s, f in SAMPLING.items():
            for kind in ("texture", "noise", "edges"):
                cases.append((f"{h}x{w}-{s}-{kind}", encode(content(kind, h, w), [cv2.IMWRITE_JPEG_QUALITY, 95,
                                                                                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR, f])))
        cases.append((f"{h}x{w}-gray", encode(content("texture", h, w), [cv2.IMWRITE_JPEG_QUALITY, 90], gray=True)))
    for q in (30, 75, 100):
        for s, f in SAMPLING.items():
            cases.append((f"q{q}-{s}", encode(content("edges", 333, 250, q), [cv2.IMWRITE_JPEG_QUALITY, q,
                                                                            cv2.IMWRITE_JPEG_SAMPLING_FACTOR, f])))
    cases.append(("luma90-chroma40", encode(content("noise", 120, 96), [cv2.IMWRITE_JPEG_LUMA_QUALITY, 90,
                                                                        cv2.IMWRITE_JPEG_CHROMA_QUALITY, 40])))
    cases.append(("dqt16", with_16bit_dqt(encode(content("edges", 61, 47), [cv2.IMWRITE_JPEG_QUALITY, 60]))))
    cases.append(("optimize", encode(content("texture", 333, 250), [cv2.IMWRITE_JPEG_OPTIMIZE, 1])))
    for r in (1, 7):
        for s, f in SAMPLING.items():
            cases.append((f"rst{r}-{s}", encode(content("edges", 100, 75, r), [cv2.IMWRITE_JPEG_RST_INTERVAL, r,
                                                                             cv2.IMWRITE_JPEG_SAMPLING_FACTOR, f])))
        cases.append((f"rst{r}-gray", encode(content("noise", 50, 41), [cv2.IMWRITE_JPEG_RST_INTERVAL, r], gray=True)))
    return cases


def orientation_cases():
    base = {"420": encode(content("texture", 37, 50), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING["420"]]),
            "gray": encode(content("edges", 37, 50), gray=True)}
    return [(f"orient{o}-{k}", with_orientation(b, o)) for o in range(1, 9) for k, b in base.items()]


def unsupported_cases():
    rgb = content("texture", 40, 56)
    return [("progressive", encode(rgb, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])),
            ("411", encode(rgb, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])),
            ("440", encode(rgb, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440]))]
