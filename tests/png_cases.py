"""PNG files for the depth-PNG decoder tests (tests/test_png_host.py, tests/test_png_gpu.py), written with cv2.imencode and
by hand (Python's zlib and struct), and cv2's result for them: the decoder's acceptance bar is byte equality with the
installed OpenCV's cv2.imdecode(IMREAD_UNCHANGED)."""
import struct
import zlib

import cv2
import numpy as np

from helpers import synth

SIZES = [(1, 1), (1, 37), (29, 1), (17, 33), (540, 720), (720, 540)]      # (h, w)
LARGE = (1080, 1920)


def content(kind, h, w, depth=16, seed=0):
    """uint16 (depth 16) or uint8 [h, w]: Map-free-like depth in millimetres (zeros included), per-pixel noise
    (literal-heavy), a constant (distance-1 / 2 copies), or a gradient."""
    rng = np.random.default_rng(seed + 7 * h + w)
    top = 65535 if depth == 16 else 255
    if kind == "depth":
        mm = np.round(synth.make_depth(rng, h, w).astype(np.float64) * 1000.0).astype(np.uint16)
        im = mm if depth == 16 else (mm // 32).astype(np.uint8)
    elif kind == "noise":
        im = rng.integers(0, top + 1, (h, w))
    elif kind == "const":
        im = np.full((h, w), 1234 % (top + 1))
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        im = (yy * 37 + xx * 11) % (top + 1)
    return np.ascontiguousarray(im.astype(np.uint16 if depth == 16 else np.uint8))


def all_values():
    """256 x 256 uint16 holding every value once."""
    return np.arange(65536, dtype=np.uint16).reshape(256, 256)


def cv2_png(im, params=()):
    ok, buf = cv2.imencode(".png", im, list(params))
    assert ok
    return buf.tobytes()


def cv2_decode(data):
    """cv2.imread(IMREAD_UNCHANGED) of the file's bytes (None where OpenCV cannot read it)."""
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)


# ------------------------------------------------------------------------------------------ hand-built files
def chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def ihdr(w, h, depth=16, color=0, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color, 0, 0, interlace))


def filter_rows(im, filters):
    """The filtered stream of a gray image: row r with filter filters[r] (0-4), samples big-endian."""
    h = im.shape[0]
    raw = im.astype(">u2").view(np.uint8).reshape(h, -1) if im.dtype == np.uint16 else im.reshape(h, -1)
    bpp = 2 if im.dtype == np.uint16 else 1
    x = raw.astype(np.int32)
    out = []
    for r in range(h):
        cur = x[r]
        up = x[r - 1] if r else np.zeros_like(cur)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]])
        ul = np.concatenate([np.zeros(bpp, np.int32), up[:-bpp]])
        f = int(filters[r])
        if f == 0:
            v = cur
        elif f == 1:
            v = cur - left
        elif f == 2:
            v = cur - up
        elif f == 3:
            v = cur - (left + up) // 2
        else:
            p = left + up - ul
            pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
            v = cur - np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
        out.append(bytes([f]) + (v & 255).astype(np.uint8).tobytes())
    return b"".join(out)


def deflate(stream, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    if not flush_every:
        return c.compress(stream) + c.flush()
    parts = [c.compress(stream[i:i + flush_every]) + c.flush(flush) for i in range(0, len(stream), flush_every)]
    return b"".join(parts) + c.flush()


def build(im, filters=None, z=None, split=0, zero_idats=False, before=(), after=(), depth=None, color=0, interlace=0):
    """A PNG of gray image `im`: row filters (default Sub), zlib stream `z` (default level 6), IDATs of `split` bytes
    (0: one), zero-length IDATs between them, extra chunks before / after the IDATs."""
    h, w = im.shape
    depth = depth or (16 if im.dtype == np.uint16 else 8)
    if z is None:
        z = deflate(filter_rows(im, [1] * h if filters is None else filters))
    pieces = [z[i:i + split] for i in range(0, len(z), split)] if split else [z]
    idats = []
    for p in pieces:
        idats.append(chunk(b"IDAT", p))
        if zero_idats:
            idats.append(chunk(b"IDAT", b""))
    return (b"\x89PNG\r\n\x1a\n" + ihdr(w, h, depth, color, interlace) + b"".join(before) + b"".join(idats) +
            b"".join(after) + chunk(b"IEND", b""))


ANCILLARY = [chunk(b"tEXt", b"Comment\x00depth in mm"), chunk(b"pHYs", struct.pack(">IIB", 2835, 2835, 1)),
             chunk(b"tIME", struct.pack(">HBBBBB", 2024, 5, 6, 7, 8, 9)), chunk(b"zTXt", b"k\x00\x00" + zlib.compress(b"v")),
             chunk(b"iTXt", b"k\x00\x00\x00\x00\x00v")]


def matrix():
    """[(name, bytes)] of supported files."""
    cases = []
    for depth in (16, 8):
        for h, w in SIZES:
            for kind in ("depth", "noise", "const", "gradient"):
                cases.append((f"{h}x{w}-{kind}-{depth}", cv2_png(content(kind, h, w, depth))))
        im = content("depth", 61, 47, depth, 5)
        for lvl in range(10):
            cases.append((f"cv2-level{lvl}-{depth}", cv2_png(im, [cv2.IMWRITE_PNG_COMPRESSION, lvl])))
        for name in ("DEFAULT", "FILTERED", "HUFFMAN_ONLY", "RLE", "FIXED"):
            cases.append((f"cv2-strategy-{name}-{depth}", cv2_png(im, [cv2.IMWRITE_PNG_STRATEGY, getattr(cv2, f"IMWRITE_PNG_STRATEGY_{name}")])))
        for name in ("FILTER_NONE", "FILTER_SUB", "FILTER_UP", "FILTER_AVG", "FILTER_PAETH", "FAST_FILTERS", "ALL_FILTERS"):
            cases.append((f"cv2-{name}-{depth}", cv2_png(im, [cv2.IMWRITE_PNG_FILTER, getattr(cv2, f"IMWRITE_PNG_{name}")])))
        # hand-built: forced and mixed filters
        im = content("depth", 40, 53, depth, 9)
        for f in range(5):
            cases.append((f"filter{f}-{depth}", build(im, [f] * 40)))
        rng = np.random.default_rng(depth)
        for k in range(2):
            cases.append((f"filter-mix{k}-{depth}", build(im, rng.integers(0, 5, 40))))
        mixed = rng.integers(0, 5, 40)
        raw = filter_rows(im, mixed)
        for lvl in (0, 1, 6, 9):
            cases.append((f"zlib-level{lvl}-{depth}", build(im, z=deflate(raw, lvl))))
        for name in ("Z_FIXED", "Z_HUFFMAN_ONLY", "Z_RLE"):
            cases.append((f"zlib-{name}-{depth}", build(im, z=deflate(raw, 6, strategy=getattr(zlib, name)))))
        for wb in range(9, 16):
            cases.append((f"wbits{wb}-{depth}", build(im, z=deflate(raw, 9, wb))))
        cases.append((f"sync-flush-{depth}", build(im, z=deflate(raw, 6, flush_every=700))))
        cases.append((f"full-flush-{depth}", build(im, z=deflate(raw, 6, flush_every=900, flush=zlib.Z_FULL_FLUSH))))
        for split in (1, 7, 8192):
            cases.append((f"split{split}-{depth}", build(im, mixed, split=split, zero_idats=split != 1)))
        cases.append((f"zero-idats-{depth}", build(im, mixed, split=256, zero_idats=True)))
        cases.append((f"ancillary-{depth}", build(im, mixed, before=ANCILLARY[:3], after=ANCILLARY[3:])))
    # stored blocks across 64 KB, and a large frame
    big = content("noise", 300, 200, 16, 3)
    cases.append(("zlib-level0-big-16", build(big, z=deflate(filter_rows(big, [0] * 300), 0))))
    cases.append(("all-values-16", cv2_png(all_values())))
    cases.append(("all-values-paeth-16", build(all_values(), [4] * 256)))
    h, w = LARGE
    cases.append((f"{h}x{w}-depth-16", cv2_png(content("depth", h, w, 16, 1))))
    # Map-free-sized depth at zlib 6 with per-row adaptive filters: literal / length codes up to 15 bits spread over
    # many root prefixes (large Huffman subtables)
    for seed in range(2):
        im = content("depth", 720, 540, 16, seed)
        cases.append((f"adaptive-zlib6-720x540-{seed}", build(im, adaptive_filters(im))))
    return cases


def adaptive_filters(im):
    """libpng's per-row heuristic: the filter whose bytes have the least sum of |signed value|."""
    streams = [filter_rows(im, [f] * im.shape[0]) for f in range(5)]
    rb = len(streams[0]) // im.shape[0]
    cost = [np.abs(np.frombuffer(st, np.int8).reshape(im.shape[0], rb)[:, 1:].astype(np.int32)).sum(1) for st in streams]
    return np.argmin(np.stack(cost), 0)


def unsupported_cases():
    g16, g8 = content("depth", 20, 24, 16), content("depth", 20, 24, 8)
    rgb = np.stack([g8, g8 // 2, 255 - g8], -1)
    return [("color2", cv2_png(rgb)), ("color6", cv2_png(np.dstack([rgb, g8]))),
            ("color4", build(g8, z=deflate(filter_rows(np.repeat(g8, 2, 1), [0] * 20)), color=4)),
            ("color3", build(g8, before=[chunk(b"PLTE", bytes(range(256)) * 3)], color=3)),
            ("depth1", cv2_png((g8 > 100).astype(np.uint8) * 255, [cv2.IMWRITE_PNG_BILEVEL, 1])),
            ("depth2", build(g8, z=deflate(b"".join(b"\x00" + bytes(6) for _ in range(20))), depth=2)),
            ("depth4", build(g8, z=deflate(b"".join(b"\x00" + bytes(12) for _ in range(20))), depth=4)),
            ("adam7", build(g16, interlace=1)),
            ("tRNS", build(g16, before=[chunk(b"tRNS", b"\x00\x00")])),
            ("sBIT", build(g16, before=[chunk(b"sBIT", b"\x0c")])),
            ("gAMA", build(g16, before=[chunk(b"gAMA", struct.pack(">I", 45455))])),
            ("eXIf", build(g16, before=[chunk(b"eXIf", b"MM\x00*\x00\x00\x00\x08\x00\x00")]))]


def _fix_crc(data, off):
    """Recomputes the CRC of the chunk at offset `off`."""
    n = int.from_bytes(data[off:off + 4], "big")
    data[off + 8 + n:off + 12 + n] = struct.pack(">I", zlib.crc32(bytes(data[off + 4:off + 8 + n])))


def _idat_offset(data):
    i = 8
    while data[i + 4:i + 8] != b"IDAT":
        i += 12 + int.from_bytes(data[i:i + 4], "big")
    return i


def malformed_cases():
    """[(name, bytes, where)]: where = "header" (mfr_png_info fails) or "decode" (the headers parse, the data fails)."""
    im = content("depth", 30, 41, 16, 2)
    raw = filter_rows(im, [1] * 30)
    good = build(im, z=deflate(raw))
    out = []
    out.append(("signature", b"\x89PNG\r\n\x1a\x0b" + good[8:], "header"))
    bad = bytearray(good); bad[8 + 8 + 3] ^= 1                                       # IHDR width, CRC not fixed
    out.append(("ihdr-crc", bytes(bad), "header"))
    bad = bytearray(good); bad[8 + 8 + 8] = 3; _fix_crc(bad, 8)                       # bit depth 3
    out.append(("ihdr-depth", bytes(bad), "header"))
    out.append(("chunk-length", good[:8 + 25] + struct.pack(">I", 1 << 31) + good[8 + 25 + 4:], "header"))
    out.append(("no-iend", good[:-12], "header"))
    out.append(("idat-before-ihdr", b"\x89PNG\r\n\x1a\n" + chunk(b"IDAT", b"") + good[8:], "header"))
    for name, hdr in (("zlib-cm", b"\x79\x9c"), ("zlib-cinfo", b"\x88\x98"), ("zlib-fcheck", b"\x78\x9d"),
                      ("zlib-fdict", b"\x78\xbb")):
        z = bytearray(deflate(raw)); z[:2] = hdr
        out.append((name, build(im, z=bytes(z)), "header"))
    # reach the device checks: corruptions with valid chunk CRCs, and one without
    bad = bytearray(good); o = _idat_offset(bad); bad[o + 8 + 40] ^= 0x10
    out.append(("idat-crc", bytes(bad), "decode"))
    z = bytearray(deflate(raw)); z[len(z) // 2] ^= 0x10
    out.append(("payload-bit", build(im, z=bytes(z)), "decode"))
    z = bytearray(deflate(raw)); z[-1] ^= 1
    out.append(("adler", build(im, z=bytes(z)), "decode"))
    z = deflate(raw)
    out.append(("truncated-stream", build(im, z=z[:len(z) * 2 // 3] + z[-4:]), "decode"))
    out.append(("extra-data", build(im, z=z[:-4] + b"\x00\x00" + z[-4:]), "decode"))
    out.append(("short-image", build(im, z=deflate(raw[:-10])), "decode"))
    out.append(("long-image", build(im, z=deflate(raw + b"\x00" * 83)), "decode"))
    bad_f = bytearray(raw); bad_f[(1 + 82) * 7] = 5
    out.append(("filter5", build(im, z=deflate(bytes(bad_f))), "decode"))
    out.append(("block-type3", build(im, z=b"\x78\x9c\x07" + z[3:]), "decode"))
    # a fixed-Huffman block whose second symbol copies from 3 bytes before the stream start
    out.append(("too-far", build(im, z=b"\x78\x01" + _fixed_too_far() + z[-4:]), "decode"))
    out.append(("beyond-window", _beyond_window(), "decode"))
    d = bytearray(good); o = _idat_offset(d); n = int.from_bytes(d[o:o + 4], "big")
    out.append(("truncated-file", bytes(d[:o + 8 + n // 2]), "header"))
    return out


def _fixed_too_far():
    """A final fixed-Huffman block: literal 0, then a match of length 3 at distance 4 (before the stream start)."""
    bits = []

    def put(v, n, rev=False):
        seq = [(v >> i) & 1 for i in range(n)]
        bits.extend(seq[::-1] if rev else seq)
    put(1, 1); put(1, 2)                      # BFINAL, BTYPE = 01
    put(0x30, 8, rev=True)                    # literal 0 (code 00110000)
    put(0b0000001, 7, rev=True)               # length 3 (symbol 257)
    put(3, 5, rev=True)                       # distance 4 (symbol 3)
    put(0, 7, rev=True)                       # end of block
    bits += [0] * (-len(bits) % 8)
    return bytes(sum(b << i for i, b in enumerate(bits[k:k + 8])) for k in range(0, len(bits), 8))


def _beyond_window():
    """A valid zlib stream whose matches reach 301 bytes back, under a header declaring a 256-byte window (CINFO 0)."""
    row = content("noise", 1, 300, 8, 4)
    im = np.repeat(row, 12, 0)
    z = bytearray(deflate(filter_rows(im, [0] * 12), 9))
    cmf = 0x08
    z[0], z[1] = cmf, (31 - (cmf * 256) % 31) % 31
    return build(im, z=bytes(z))
