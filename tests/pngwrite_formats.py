"""PNG writer and numpy pixel model for every format of the all-formats decode (FPNGB_PNG_ALL_FORMATS): palette, 1/2/4/8/16-bit
gray, 8/16-bit gray+alpha, RGB and RGBA, tRNS color keys and palette alpha, Adam7 interlacing, every row filter and nonzero padding
bits at the end of sub-byte rows.  Built from numpy and zlib only; test_decode_png_formats_cpu.py pins the model against PIL,
torchvision (libpng) and, where they are built, lodepng and wuffs."""
from __future__ import annotations

import struct
import zlib

import numpy as np

from pngwrite import IEND, SIG, chunk, ihdr, paeth

SAMPLES = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}                       # color type -> samples per pixel
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]   # x0, y0, dx, dy


def passes(w, h, interlace):
    """[(x0, y0, dx, dy, pw, ph)] of the non-empty passes"""
    out = []
    for (x0, y0, dx, dy) in (ADAM7 if interlace else [(0, 0, 1, 1)]):
        pw, ph = max(0, (w - x0 + dx - 1) // dx), max(0, (h - y0 + dy - 1) // dy)
        if pw and ph:
            out.append((x0, y0, dx, dy, pw, ph))
    return out


def raw_len(w, h, bits, interlace):
    return sum(ph * (1 + (pw * bits + 7) // 8) for (_, _, _, _, pw, ph) in passes(w, h, interlace))


def pack_rows(s: np.ndarray, depth: int, pad_rs=None) -> np.ndarray:
    """rows of samples s [ph, pw, spp] as PNG bytes [ph, rowbytes]; the padding bits of sub-byte rows are random when pad_rs is given"""
    ph, pw, spp = s.shape
    if depth == 16:
        return s.astype(">u2").view(np.uint8).reshape(ph, pw * spp * 2)
    if depth == 8:
        return s.astype(np.uint8).reshape(ph, pw * spp)
    bits = ((s.reshape(ph, pw * spp)[..., None].astype(np.uint32) >> np.arange(depth - 1, -1, -1)) & 1).reshape(ph, -1)
    nb = (bits.shape[1] + 7) // 8 * 8
    pad = np.zeros((ph, nb - bits.shape[1]), np.uint32)
    if pad_rs is not None:
        pad = pad_rs.randint(0, 2, pad.shape).astype(np.uint32)
    return np.packbits(np.concatenate([bits, pad], 1).astype(np.uint8), axis=1)


def filter_bytes(rows: np.ndarray, bpp: int, filters) -> bytes:
    """filtered scanlines of byte rows [ph, rb], filter unit bpp bytes, row y with filters[y]"""
    ph, rb = rows.shape
    out = np.zeros((ph, rb + 1), np.uint8)
    prev = np.zeros(rb, np.int32)
    z = np.zeros(bpp, np.int32)
    for y in range(ph):
        cur, ft = rows[y].astype(np.int32), int(filters[y])
        a = np.concatenate([z, cur[:-bpp]])[:rb]
        c = np.concatenate([z, prev[:-bpp]])[:rb]
        pred = [0 * cur, a, prev, (a + prev) // 2, paeth(a, prev, c)][ft]
        out[y, 0] = ft
        out[y, 1:] = (cur - pred) & 255
        prev = cur
    return out.tobytes()


def raw_stream(s: np.ndarray, ctype: int, depth: int, interlace=0, filters="random", seed=0, pad_bits=True) -> bytes:
    """the inflated bytes of samples s [h, w, spp]: every pass's filtered rows"""
    h, w, _ = s.shape
    rs = np.random.RandomState(seed)
    bits = depth * SAMPLES[ctype]
    out = b""
    for (x0, y0, dx, dy, pw, ph) in passes(w, h, interlace):
        rows = pack_rows(s[y0::dy, x0::dx], depth, rs if pad_bits else None)
        ft = rs.randint(0, 5, ph) if filters == "random" else np.full(ph, int(filters))
        out += filter_bytes(rows, max(1, bits // 8), ft)
    return out


def make_png(s: np.ndarray, ctype: int, depth: int, interlace=0, plte=None, trns=None, filters="random", seed=0, level=6,
             pad_bits=True, z=None, before=(), after=()) -> bytes:
    """a PNG of samples s [h, w, spp] (palette indices for color type 3); plte: [n, 3] uint8; trns: bytes of the tRNS chunk"""
    h, w, _ = s.shape
    if z is None:
        z = zlib.compress(raw_stream(s, ctype, depth, interlace, filters, seed, pad_bits), level)
    body = list(before)
    if plte is not None:
        body.append(chunk(b"PLTE", np.asarray(plte, np.uint8).tobytes()))
    if trns is not None:
        body.append(chunk(b"tRNS", bytes(trns)))
    return SIG + ihdr(w, h, depth, ctype, interlace=interlace) + b"".join(body) + chunk(b"IDAT", z) + b"".join(after) + IEND


def key_trns(ctype: int, key) -> bytes:
    """the tRNS chunk data of a color key (type 0: one 16-bit value, type 2: three)"""
    return struct.pack(">H", key) if ctype == 0 else struct.pack(">HHH", *key)


def random_samples(rs, w, h, ctype, depth, n_plte=256):
    spp = SAMPLES[ctype]
    hi = (n_plte if ctype == 3 and n_plte < (1 << depth) else 1 << depth)
    return rs.randint(0, hi, (h, w, spp)).astype(np.uint32)


# ---- the pixel model (include/fpng_b200.h's rules) --------------------------------------------------------------------------------
def model16(s: np.ndarray, ctype: int, depth: int, plte=None, trns=None) -> np.ndarray:
    """[h, w, 4] RGBA in the 16-bit domain: 16-bit samples as they are, 8-bit values v as v * 257, missing alpha 0xFFFF"""
    s = s.astype(np.int64)
    h, w, _ = s.shape
    mul = 1 if depth == 16 else 257
    full = np.full((h, w), 0xFFFF, np.int64)
    if ctype == 3:
        n = len(plte)
        pal = np.zeros((256, 4), np.int64)
        pal[:, 3] = 255
        pal[:n, :3] = np.asarray(plte, np.int64)
        if trns is not None:
            t = np.frombuffer(bytes(trns), np.uint8).astype(np.int64)
            pal[:len(t), 3] = t
        return pal[s[..., 0]] * 257
    if ctype in (0, 4):
        y = s[..., 0] * (255 // ((1 << depth) - 1) * 257 if depth < 8 else mul)
        if ctype == 4:
            a = s[..., 1] * mul
        elif trns is not None:
            a = np.where(s[..., 0] == struct.unpack(">H", bytes(trns))[0], 0, full)
        else:
            a = full
        return np.stack([y, y, y, a], -1)
    rgb = s[..., :3] * mul
    if ctype == 6:
        a = s[..., 3] * mul
    elif trns is not None:
        key = np.array(struct.unpack(">HHH", bytes(trns)), np.int64)
        a = np.where((s[..., :3] == key).all(-1), 0, full)
    else:
        a = full
    return np.concatenate([rgb, a[..., None]], -1)


def model_u8(s, ctype, depth, desired, plte=None, trns=None) -> np.ndarray:
    return (model16(s, ctype, depth, plte, trns)[..., :desired] >> 8).astype(np.uint8)


def model_values(s, ctype, depth, desired, plte=None, trns=None) -> np.ndarray:
    """float32 v of the typed output: s / 257 (correctly rounded) for 16-bit files, the uint8 value otherwise"""
    m = model16(s, ctype, depth, plte, trns)[..., :desired]
    if depth == 16:
        return m.astype(np.float32) / np.float32(257.0)
    return (m >> 8).astype(np.float32)


def info_chans(ctype: int, trns) -> int:
    base = {0: 1, 2: 3, 3: 3, 4: 2, 6: 4}[ctype]
    return base + (1 if trns is not None and ctype in (0, 2, 3) else 0)


def case(rs, w, h, ctype, depth, interlace=0, with_trns=False, filters="random", seed=0, n_plte=None):
    """(png, samples, plte, trns): random samples; palettes of n_plte (default random) entries; tRNS a color key that some pixels
    hit, or a random palette alpha table"""
    plte = trns = None
    if ctype == 3:
        n = n_plte or int(rs.randint(1, (1 << depth) + 1))
        plte = rs.randint(0, 256, (n, 3)).astype(np.uint8)
        s = random_samples(rs, w, h, ctype, depth, n)
        if with_trns:
            trns = rs.randint(0, 256, int(rs.randint(0, n + 1))).astype(np.uint8).tobytes()
    else:
        s = random_samples(rs, w, h, ctype, depth)
        if with_trns:
            px = s[int(rs.randint(0, h)), int(rs.randint(0, w))]
            trns = key_trns(ctype, int(px[0]) if ctype == 0 else [int(v) for v in px[:3]])
    png = make_png(s, ctype, depth, interlace, plte, trns, filters, seed)
    return png, s, plte, trns


def combos():
    """every (color type, depth, interlace, tRNS) combination the all-formats decode reads (tRNS only in types 0 / 2 / 3)"""
    out = []
    for ctype, depths in DEPTHS.items():
        for depth in depths:
            for interlace in (0, 1):
                for t in ((False, True) if ctype in (0, 2, 3) else (False,)):
                    out.append((ctype, depth, interlace, t))
    return out


# ---- a reader for files other writers produced (PIL, OpenCV): samples, palette and tRNS as the model takes them ------------------
def _unfilter_run(f: np.ndarray, ft: np.ndarray, prev: np.ndarray, bpp: int) -> np.ndarray:
    """rows of a run of None / Sub / Up rows at once: None and Sub rows stand alone, an Up row adds the row above, so each row
    is the last stand-alone row at or above it (or prev) plus the Up rows' bytes since"""
    n, rb = f.shape
    own = f.copy()
    sub = ft == 1
    if sub.any():
        own[sub] = np.cumsum(f[sub].reshape(int(sub.sum()), rb // bpp, bpp), 1).reshape(-1, rb)
    up = ft == 2
    c = np.cumsum(np.where(up[:, None], f, 0), 0)
    anchor = np.maximum.accumulate(np.where(up, -1, np.arange(n)))
    a = np.maximum(anchor, 0)
    start = np.where(anchor[:, None] >= 0, own[a] - c[a], prev[None, :])
    return (start + c) & 255


def _unfilter(raw: np.ndarray, rb: int, ph: int, bpp: int) -> np.ndarray:
    buf = raw.reshape(ph, rb + 1).astype(np.int64)
    out = np.zeros((ph, rb), np.int64)
    prev = np.zeros(rb, np.int64)
    fts = buf[:, 0]
    assert (fts <= 4).all()
    y = 0
    while y < ph:
        if fts[y] <= 2:                                                # the run of None / Sub / Up rows from y
            e = y
            while e < ph and fts[e] <= 2:
                e += 1
            out[y:e] = _unfilter_run(buf[y:e, 1:], fts[y:e], prev, bpp)
            prev = out[e - 1]
            y = e
            continue
        ft, f = int(fts[y]), buf[y, 1:]
        if ft in (0, 2):
            cur = (f + (prev if ft == 2 else 0)) & 255
        elif ft == 1:
            cur = (np.cumsum(f.reshape(-1, bpp), 0) & 255).reshape(-1)
        else:
            cur = np.zeros(rb, np.int32)
            for x in range(rb):
                a = cur[x - bpp] if x >= bpp else 0
                c = prev[x - bpp] if x >= bpp else 0
                cur[x] = (f[x] + ((a + prev[x]) // 2 if ft == 3 else int(paeth(np.int32(a), np.int32(prev[x]), np.int32(c))))) & 255
        out[y] = cur
        prev = cur
        y += 1
    return out.astype(np.uint8)


def parse(data: bytes) -> dict:
    """{w, h, ctype, depth, interlace, samples [h, w, spp], plte [n, 3] or None, trns bytes or None}"""
    pos, idat, plte, trns = 8, b"", None, None
    w, h, depth, ctype, _, _, il = struct.unpack(">IIBBBBB", data[16:29])
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if tag == b"IDAT":
            idat += body
        elif tag == b"PLTE":
            plte = np.frombuffer(body, np.uint8).reshape(-1, 3)
        elif tag == b"tRNS" and ctype in (0, 2, 3):
            trns = body
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8)
    spp, at = SAMPLES[ctype], 0
    bits = depth * spp
    s = np.zeros((h, w, spp), np.uint32)
    for (x0, y0, dx, dy, pw, ph) in passes(w, h, il):
        rb = (pw * bits + 7) // 8
        rows = _unfilter(raw[at:at + ph * (rb + 1)], rb, ph, max(1, bits // 8))
        at += ph * (rb + 1)
        if depth == 16:
            v = rows.view(">u2").reshape(ph, pw, spp)
        elif depth == 8:
            v = rows.reshape(ph, pw, spp)
        else:
            b = np.unpackbits(rows, axis=1)[:, :pw * depth].reshape(ph, pw, depth)
            v = (b.astype(np.uint32) << np.arange(depth - 1, -1, -1, dtype=np.uint32)).sum(-1).reshape(ph, pw, 1)
        s[y0::dy, x0::dx] = v
    return {"w": w, "h": h, "ctype": ctype, "depth": depth, "interlace": il, "samples": s, "plte": plte, "trns": trns}
