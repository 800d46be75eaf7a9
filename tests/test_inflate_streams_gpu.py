"""Differential tests of the any-PNG inflate (png_inflate_kernel) on Deflate streams zlib never writes: tests/deflategen.py's
block plans (stored / fixed / dynamic, empty blocks, codes of up to 15 bits, code-length runs across the lit/dist boundary,
distance 32768 and matches back to byte 0), its named invalid streams, and a few thousand seeded mutants of its streams, each
judged by zlib (deflategen.expect) rather than by the writer.  Pixels of big accepted mutants are compared with a partner file of
the same IHDR whose stream zlib wrote from the expected bytes, so no Python unfilter runs on them."""
import functools
import struct
import zlib

import numpy as np
import pytest

import deflategen as dg
import pngwrite
import pngwrite_formats as pf
import test_decode_png_formats_gpu as fmt
from pngwrite import COLOR_TYPE, IEND, SIG, chunk, ihdr
from test_decode_png_gpu import ADLER, GUARD, INVALID_IDAT, PENDING, run

pytestmark = pytest.mark.gpu


def idat_split(z: bytes, rs) -> list:
    """IDAT payloads: random cut points, some chunks tiny or empty"""
    cuts = sorted(set(int(c) for c in rs.randint(0, len(z) + 1, int(rs.randint(0, 6)) + len(z) // 20000)))
    parts = [z[a:b] for a, b in zip([0] + cuts, cuts + [len(z)])]
    return [p for p in parts if p or rs.randint(0, 3) == 0] or [b""]


def png8(w, h, c, z, seed) -> bytes:
    rs = np.random.RandomState(seed)
    return SIG + ihdr(w, h, ctype=COLOR_TYPE[c]) + b"".join(chunk(b"IDAT", p) for p in idat_split(z, rs)) + IEND


def resplit(png: bytes, seed) -> bytes:
    """png with its IDAT run cut again at random points"""
    pos, head, z, tail = 8, b"", b"", b""
    while pos < len(png):
        n = struct.unpack(">I", png[pos:pos + 4])[0]
        c = png[pos:pos + 12 + n]
        if c[4:8] == b"IDAT":
            z += c[8:8 + n]
        elif z:
            tail += c
        else:
            head += c
        pos += 12 + n
    return SIG + head + b"".join(chunk(b"IDAT", p) for p in idat_split(z, np.random.RandomState(seed))) + tail


def views_np(raw, st, info, oo, d):
    r = raw.cpu().numpy()
    return [r[int(oo[k]):int(oo[k]) + int(info[k][1]) * int(info[k][2]) * d].reshape(int(info[k][2]), int(info[k][1]), d)
            if st[k] == 0 else None for k in range(len(st))], r


def check_guards(r, st, info, oo, d):
    """no byte outside the decoded files' outputs was written, and no status was left pending"""
    mask = np.ones(r.size, bool)
    for k in range(len(st)):
        if st[k] == 0:
            mask[int(oo[k]):int(oo[k]) + int(info[k][1]) * int(info[k][2]) * d] = False
    assert (r[mask] == GUARD).all()
    assert not (st == PENDING).any()


def with_verify(gpu, on, fn):
    gpu.set_decode_verify(on)
    try:
        return fn()
    finally:
        gpu.set_decode_verify(False)


def model(raw, w, h, c):
    img = pngwrite.unfilter(raw, w, h, c)
    assert img is not None
    return img


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("d", [3, 4])
def test_valid_corpus(gpu, d, verify):
    cases = dg.corpus()
    files = [png8(w, h, c, s.z, k) for k, (w, h, c, raw, s) in enumerate(cases)]
    views, st, info, oo, raw = with_verify(gpu, verify, lambda: run(gpu, files, d))
    vs, r = views_np(raw, st, info, oo, d)
    check_guards(r, st, info, oo, d)
    for k, img in enumerate(corpus_model()):
        assert st[k] == 0, (k, st[k])
        np.testing.assert_array_equal(vs[k], pngwrite.expand(img, d), err_msg=str(img.shape))


@functools.lru_cache(maxsize=None)
def corpus_model():
    return [model(raw, w, h, c) for (w, h, c, raw, _) in dg.corpus()]


def ext_files():
    return [(resplit(pf.make_png(s, ctype, depth, il, plte, z=st.z), k), s, ctype, depth, plte)
            for k, (s, ctype, depth, il, plte, raw, st) in enumerate(dg.ext_corpus())]


@pytest.mark.parametrize("verify", [False, True])
def test_ext_files(gpu, verify):
    """palette 2-bit Adam7 and 16-bit RGB: the inflate's length is PngDesc::raw_len"""
    cases = ext_files()
    for d in (3, 4):
        views, st, _, _ = with_verify(gpu, verify, lambda: fmt.run(gpu, [c[0] for c in cases], d))
        for k, (png, s, ctype, depth, plte) in enumerate(cases):
            assert st[k] == 0, (k, st[k])
            np.testing.assert_array_equal(views[k].cpu().numpy(), pf.model_u8(s, ctype, depth, d, plte), err_msg=str(k))


def invalid_8bit():
    out = []
    for k, (w, h, c, raw, _) in enumerate(dg.corpus()[3:7]):
        out += [(name, png8(w, h, c, z, k)) for name, z in dg.invalid_streams(raw, 50 + k).items()]
    return out


def invalid_ext():
    out = []
    for k, (s, ctype, depth, il, plte, raw, _) in enumerate([dg.ext_corpus()[i] for i in (0, 1, 3, 5)]):
        out += [(name, resplit(pf.make_png(s, ctype, depth, il, plte, z=z), k)) for name, z in dg.invalid_streams(raw, 60 + k).items()]
    return out


@pytest.mark.parametrize("verify", [False, True])
def test_invalid_corpus(gpu, verify):
    cases = invalid_8bit()
    views, st, info, oo, raw = with_verify(gpu, verify, lambda: run(gpu, [c[1] for c in cases], 4))
    _, r = views_np(raw, st, info, oo, 4)
    bad = [(name, int(s)) for (name, _), s in zip(cases, st) if s != INVALID_IDAT]
    assert not bad, bad
    assert (r == GUARD).all()
    ext = invalid_ext()
    _, st, _, r = with_verify(gpu, verify, lambda: fmt.run(gpu, [c[1] for c in ext], 4))
    bad = [(name, int(s)) for (name, _), s in zip(ext, st) if s != INVALID_IDAT]
    assert not bad, bad
    assert (r.cpu().numpy() == GUARD).all()


# ---- mutation fuzz ----------------------------------------------------------------------------------------------------------
def mutate(rs, s: dg.Stream) -> bytes:
    z = bytearray(s.z)
    kind = int(rs.randint(0, 7))
    if kind == 0:                                                       # bit flip
        p = int(rs.randint(0, len(z)))
        z[p] ^= 1 << int(rs.randint(0, 8))
    elif kind == 1:                                                     # byte overwrite
        z[int(rs.randint(0, len(z)))] = int(rs.randint(0, 256))
    elif kind == 2:                                                     # truncation
        z = z[:int(rs.randint(0, len(z)))]
    elif kind == 3:                                                     # insertion
        p = int(rs.randint(0, len(z) + 1))
        z[p:p] = bytes([int(rs.randint(0, 256))])
    elif kind == 4:                                                     # deletion
        del z[int(rs.randint(0, len(z)))]
    elif kind == 5:                                                     # a flipped BTYPE bit
        t, at, _ = s.blocks[int(rs.randint(0, len(s.blocks)))]
        b = at + 1 + int(rs.randint(0, 2))
        z[b >> 3] ^= 1 << (b & 7)
    else:                                                               # stored LEN / NLEN edited, with or without NLEN kept
        stored = [b for b in s.blocks if b[0] == 0]
        if not stored:
            return mutate(rs, s)
        at = stored[int(rs.randint(0, len(stored)))][2]
        n = struct.unpack("<H", z[at:at + 2])[0]
        m = (n + int(rs.choice([-2, -1, 1, 2, 1000, 40000]))) & 0xFFFF
        z[at:at + 2] = struct.pack("<H", m)
        if rs.randint(0, 2):
            z[at + 2:at + 4] = struct.pack("<H", m ^ 0xFFFF)
    return bytes(z)


def fuzz_items():
    """[(png, w, h, c, expected status verify off, verify on, expected raw or None, partner index)]: mutants, then partners"""
    rs = np.random.RandomState(11)
    items, partners = [], []
    for b, (w, h, c, raw, s) in enumerate(dg.fuzz_bases()):
        for m in range(120):
            z = mutate(rs, s)
            e = dg.expect(z, len(raw))
            stride = w * c + 1
            if e is None or max(e[0][::stride]) > 4:
                items.append((png8(w, h, c, z, m), w, h, c, INVALID_IDAT, INVALID_IDAT, None, -1))
                continue
            out, adler = e
            part = len(partners)
            partners.append((png8(w, h, c, zlib.compress(out, 1), m + 1), w, h, c, 0, 0, out, -1))
            items.append((png8(w, h, c, z, m), w, h, c, 0, 0 if adler == "ok" else ADLER, out, part))
    n = len(items)
    return [it[:7] + (it[7] + n if it[7] >= 0 else -1,) for it in items] + partners


@pytest.fixture(scope="module")
def fuzz():
    return fuzz_items()


def check_fuzz(res, items, verify, d=4):
    views, st, info, oo, raw = res
    vs, r = views_np(raw, st, info, oo, d)
    check_guards(r, st, info, oo, d)
    want = np.array([it[5] if verify else it[4] for it in items])
    bad = np.nonzero(st != want)[0]
    assert bad.size == 0, [(int(k), int(st[k]), int(want[k])) for k in bad[:20]]
    for k, (png, w, h, c, _, _, out, part) in enumerate(items):
        if st[k] != 0 or part < 0:
            continue
        np.testing.assert_array_equal(vs[k], vs[part], err_msg=str(k))
        if len(out) <= 20000:
            np.testing.assert_array_equal(vs[k], pngwrite.expand(model(out, w, h, c), d), err_msg=str(k))
    return vs


def test_mutation_fuzz(gpu, fuzz):
    files = [it[0] for it in fuzz]
    assert len(files) > 2000 and sum(1 for it in fuzz if it[4] == 0) > 200
    first = check_fuzz(run(gpu, files, 4, rs=np.random.RandomState(1)), fuzz, False)
    check_fuzz(with_verify(gpu, True, lambda: run(gpu, files, 4, rs=np.random.RandomState(2))), fuzz, True)
    # the same files in another order at other offsets: statuses and pixels do not depend on what the workspace held before
    order = np.random.RandomState(3).permutation(len(files))
    views, st, info, oo, raw = run(gpu, [files[i] for i in order], 4, rs=np.random.RandomState(4))
    vs, _ = views_np(raw, st, info, oo, 4)
    for j, i in enumerate(order):
        assert st[j] == fuzz[i][4], (int(i), int(st[j]))
        if st[j] == 0:
            assert np.array_equal(vs[j], first[i]), int(i)


# ---- fpng files without fdEC: a second encoder's streams through the general path ------------------------------------------------
def drop_fdec(png: bytes) -> bytes:
    pos, out = 8, [png[:8]]
    while pos < len(png):
        n = struct.unpack(">I", png[pos:pos + 4])[0]
        if png[pos + 4:pos + 8] != b"fdEC":
            out.append(png[pos:pos + 12 + n])
        pos += 12 + n
    return b"".join(out)


def test_fpng_without_fdec(gpu):
    import imagegen
    files = []
    for k, (w, h, c) in enumerate([(5, 3, 3), (300, 200, 3), (257, 129, 4), (1000, 700, 3), (640, 480, 4)]):
        img = imagegen.make(("g1", "g0", "runs")[k % 3], w, h, c, k)
        for flags in (0, 1, 2):                                         # 1-pass, FPNG_ENCODE_SLOWER, FPNG_FORCE_UNCOMPRESSED
            ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c, flags)
            assert ok
            files.append(png)
    general = [drop_fdec(f) for f in files]
    assert all(len(g) < len(f) for g, f in zip(general, files))
    for d in (3, 4):
        ref, ref_st, _, _, _ = run(gpu, files, d, any_png=False)
        got, st, _, _, _ = run(gpu, general, d)
        assert (ref_st == 0).all() and (st == 0).all(), (ref_st, st)
        for k in range(len(files)):
            assert np.array_equal(got[k].cpu().numpy(), ref[k].cpu().numpy()), k
