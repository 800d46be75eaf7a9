"""GPU tests of the resized and native decodes at their tile, tap-count, CTA-width and 4 GiB edges (cases: tests/decode_edges.py).

Resized outputs are compared with decode_edges' float64 model within its error bound E: float outputs within E * |scale| plus the
rounding of the division by 257, of the scale and bias and of the output type; uint8 and uint16 outputs equal to a rounding of some
value in [r - E, r + E].  Outputs too large for the host are compared on a seeded sample of whole rows.  Native ragged outputs
are compared exactly with test_decode_native_cpu's model.  Cases that need more than 4 GB of device memory skip themselves
unless three times their need is free."""
import numpy as np
import pytest

import decode_edges as de
import pngwrite_formats as pf
from test_decode_native_cpu import fpng_native16, native16, native_out
from test_decode_native_gpu import as_np, packed

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
STATS = {}


@pytest.fixture(autouse=True)
def _peak_memory():
    """prints each test's peak of torch's allocator and the device memory in use after it, which includes the decode workspace
    (the library allocates it itself and keeps it): the figures the skip rules of the 4 GiB cases are based on"""
    import torch
    torch.cuda.reset_peak_memory_stats()
    yield
    free, total = torch.cuda.mem_get_info()
    print("torch peak %.2f GB, device in use after %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9, (total - free) / 1e9))


def need_free(gb):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * gb * 1e9:
        pytest.skip(f"needs {gb} GB of device memory and three times that free; {free / 1e9:.1f} GB free")


def record(family, got, r, E):
    """the largest |got - r| of a family and its ratio to E (float32 outputs at scale 1, bias 0, where got - r is the resize's own
    error)"""
    d = np.abs(got - r)
    m, q = STATS.get(family, (0.0, 0.0))
    STATS[family] = (max(m, float(d.max())), max(q, float((d / E).max())))
    print(family, "max |got - r| %.3g, max ratio to E %.3f" % STATS[family])


def rne(v, top):
    return np.clip(np.round(v), 0, top)                                          # numpy rounds half to even, as cvt.rni


def check(got, r, E, dtype, native, s=None, b=None):
    """got [.., C] as float64, r the model's values and E the bound (both in the resize's domain: 0..255, or 0..65535 native)"""
    E = np.broadcast_to(E, r.shape)
    if dtype == "uint16":
        assert native
        bad = (got < rne(r - E, 65535)) | (got > rne(r + E, 65535))
        assert not bad.any(), (np.argwhere(bad)[:4], got[bad][:4], r[bad][:4], E[bad][:4])
        return
    if native:                                   # v = fl(o / 257): one more rounding
        r, E = r / 257.0, E / 257.0 + U * (np.abs(r) + E) / 257.0
    if dtype == "uint8":
        bad = (got < rne(r - E, 255)) | (got > rne(r + E, 255))
        assert not bad.any(), (np.argwhere(bad)[:4], got[bad][:4], r[bad][:4])
        return
    s = np.ones(got.shape[-1]) if s is None else np.asarray(s, np.float64)
    b = np.zeros(got.shape[-1]) if b is None else np.asarray(b, np.float64)
    w = r * s + b
    tol = E * np.abs(s) + 2 * U * (np.abs(r * s) + np.abs(w) + E * np.abs(s))
    if dtype != "float32":
        from test_decode_resized_gpu import ulp
        import torch
        tol = tol + ulp(getattr(torch, dtype), w)
    d = np.abs(got - w)
    assert (d <= tol).all(), (np.argwhere(d > tol)[:4], got[d > tol][:4], w[d > tol][:4], tol[d > tol][:4])


def resize(gpu, files, d, size, dtype, native, aa, boxes=None, scale=None, bias=None):
    """one resized call into an [n, H, W, d] output (guard-filled); returns the device output"""
    import torch
    data, offsets, sizes = packed(files)
    T = getattr(torch, dtype)
    out = torch.empty((len(files),) + tuple(size) + (d,), dtype=T, device="cuda")
    out.view(torch.uint8).fill_(0xA5)
    bx = None if boxes is None else torch.from_numpy(np.asarray(boxes, np.int32)).cuda()
    _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, size, d, boxes=bx, antialias=aa, out=out, scale=scale, bias=bias,
                                                any_png=True, all_formats=True, native=native)
    assert not st.any().item(), st.cpu().numpy()
    return out


def rows_of(out, f, rows):
    import torch
    idx = torch.as_tensor(np.asarray(rows), device="cuda")
    if out.dtype == torch.uint16:                                     # no uint16 indexing kernel in torch: index the int16 view
        return out.view(torch.int16)[f, idx].cpu().numpy().view(np.uint16).astype(np.float64)
    return out[f, idx].float().cpu().numpy().astype(np.float64)


def compare(out, f, fetch, crop_hw, size, aa, dtype, native, m, rows=None, family=None, s=None, b=None, col_chunk=1 << 21):
    """file f of a resized output against the model on `rows` (default all), in column chunks"""
    bh, bw = crop_hw
    H, W = size
    rows = np.arange(H) if rows is None else np.asarray(rows)
    got = rows_of(out, f, rows)
    for c0 in range(0, W, col_chunk):
        cols = np.arange(c0, min(W, c0 + col_chunk))
        r = de.model_rows(fetch, bh, bw, H, W, aa, rows, cols)
        nx, ny = de.taps(bh, bw, H, W, aa, rows, cols)
        E = de.bound(nx[None, :, None], ny[:, None, None], m)
        g = got[:, cols]
        check(g, r, E, dtype, native, s, b)
        if family and dtype == "float32" and s is None:
            record(family, g * (257.0 if native else 1.0), r, E)


def source(h, w, chans, native, seed):
    """(png, model values [h, w, chans]) of a general PNG with random filters: 8-bit RGB / RGBA, or 16-bit gray / RGBA (native)"""
    if native:
        ctype = 0 if chans == 1 else 6
        s = de.smooth(h, w, pf.SAMPLES[ctype], seed, depth=16)
        return pf.make_png(s, ctype, 16, seed=seed), native16(s, ctype, 16, chans)
    ctype = 2 if chans == 3 else 6
    s = de.smooth(h, w, chans, seed)
    return pf.make_png(s, ctype, 8, seed=seed), s.astype(np.int64)


# ---- 1. resize at scale ------------------------------------------------------------------------------------------------------
TILE_VARIANTS = [("uint8", 3, False), ("float32", 4, False), ("bfloat16", 3, False), ("uint16", 1, True), ("uint16", 4, True),
                 ("float32", 1, True)]


@pytest.mark.parametrize("variant", TILE_VARIANTS, ids=lambda v: "%s_d%d%s" % (v[0], v[1], "_native" if v[2] else ""))
def test_tile_loop(gpu, variant):
    """outputs of 524 288 and 65 792 tiles: the tile loop runs past gridDim.x, and the 2^24-wide output reaches indices >= 2^23"""
    dtype, d, native = variant
    sb = dict(scale=[0.5, 2.0, 1.0, 0.25][:d], bias=[1.0, -3.0, 0.0, 0.5][:d]) if dtype == "bfloat16" else {}
    for k, c in enumerate(de.tile_loop_cases()):
        png, px = source(c.src[0], c.src[1], d, native, 10 + k)
        out = resize(gpu, [png], d, c.out, dtype, native, c.aa, **sb)
        compare(out, 0, de.array_fetch(px), c.src, c.out, c.aa, dtype, native, int(px.max()), rows=c.rows, family="tile_loop",
                s=sb.get("scale"), b=sb.get("bias"))
        del out


def _group(cases):
    g = {}
    for c in cases:
        g.setdefault((c.out, c.aa, c.box is None), []).append(c)
    return g


@pytest.mark.parametrize("dtype", ["float32", "uint8"])
def test_tap_counts(gpu, dtype):
    """thousands of taps per output (3840 x 8, 8 x 2160, 16384 x 2 to one pixel), whole and cropped, antialias on and off"""
    srcs = {}
    for (size, aa, whole), cases in _group(de.tap_cases()).items():
        for c in cases:
            if c.src not in srcs:
                srcs[c.src] = source(c.src[0], c.src[1], 3, False, c.src[0] + c.src[1])
        out = resize(gpu, [srcs[c.src][0] for c in cases], 3, size, dtype, False, aa, None if whole else [c.box for c in cases])
        for f, c in enumerate(cases):
            px = srcs[c.src][1]
            compare(out, f, de.array_fetch(px, c.box), c.crop[2:], size, aa, dtype, False, int(px.max()), family="taps")


@pytest.mark.parametrize("dtype", ["uint16", "float32"])
def test_native_tap_counts(gpu, dtype):
    """16-bit sources at large tap counts: gray16 4096 x 16 to one pixel, RGBA16 1024 x 1024 to 3 x 3"""
    for c in de.native_tap_cases():
        png, px = source(c.src[0], c.src[1], c.chans, True, c.chans)
        out = resize(gpu, [png], c.chans, c.out, dtype, True, c.aa, None if c.box is None else [c.box])
        compare(out, 0, de.array_fetch(px, c.box), c.crop[2:], c.out, c.aa, dtype, True, int(px.max()), family="native_taps")


@pytest.fixture(scope="module")
def fpng_4k(oracle):
    import imagegen
    img = imagegen.gradient_noise(3840, 2160, 3, 5)
    return oracle.encode(img, 3840, 2160, 3, 0), img.astype(np.int64)


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_crops_fpng_4k(gpu, fpng_4k, dtype):
    """1 x 1 boxes at each corner, boxes ending on the last row, the full image minus one row and column; up- and downscaled"""
    png, px = fpng_4k
    for (size, aa, _), cases in _group(de.crop_cases(2160, 3840)).items():
        out = resize(gpu, [png] * len(cases), 3, size, dtype, False, aa, [c.box for c in cases])
        for f, c in enumerate(cases):
            compare(out, f, de.array_fetch(px, c.box), c.crop[2:], size, aa, dtype, False, 255, family="crops")


@pytest.mark.parametrize("dtype", ["uint16", "float32"])
def test_crops_16_bit(gpu, dtype):
    h, w = 1000, 1000
    s = de.smooth(h, w, 3, 6, depth=16)
    png, px = pf.make_png(s, 2, 16, seed=6), native16(s, 2, 16, 3)
    for (size, aa, _), cases in _group(de.crop_cases(h, w, native=True)).items():
        out = resize(gpu, [png] * len(cases), 3, size, dtype, True, aa, [c.box for c in cases])
        for f, c in enumerate(cases):
            compare(out, f, de.array_fetch(px, c.box), c.crop[2:], size, aa, dtype, True, int(px.max()), family="crops_16")


@pytest.fixture(scope="module")
def big_file(gpu):
    """the 24000 x 23000 RGB image of decode_edges.big_pixel, generated on the device and written by the GPU fpng encoder; returns
    the file as (data, offsets, sizes) on the device"""
    import torch
    need_free(12)
    torch.cuda.reset_peak_memory_stats()
    H, W = de.BIG_H, de.BIG_W
    img = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    x = torch.arange(W, dtype=torch.int32, device="cuda")[None, :]
    for y0 in range(0, H, 1024):
        y = torch.arange(y0, min(H, y0 + 1024), dtype=torch.int32, device="cuda")[:, None]
        base = x * 3 + y * 7 + ((x ^ y) >> 4) * 29
        for c in range(3):
            img[y0:y0 + y.shape[0], :, c] = ((base + c * 85) & 255).to(torch.uint8)
    assert gpu.max_encoded_size(W, H, 3) == 1656149430
    data, offsets, sizes = gpu.encode_png_device([img])
    del img
    n = int(sizes[0].item())
    o = int(offsets[0].item())
    buf = torch.zeros((n + 15) // 16 * 16, dtype=torch.uint8, device="cuda")
    buf[:n] = data[o:o + n]
    del data
    torch.cuda.empty_cache()
    print("big file %d bytes, peak device memory while writing it %.2f GB" % (n, torch.cuda.max_memory_allocated() / 1e9))
    return buf, torch.zeros(1, dtype=torch.int64, device="cuda"), torch.full((1,), n, dtype=torch.int32, device="cuda")


def test_big_resized_rows_past_4_gib(gpu, big_file):
    """a 64 x 48 box at the bottom-right of the 24000 x 23000 file, whose source rows start 4.4 GB into the uint16 intermediate,
    and a top-left control box"""
    import torch
    for c in de.big_cases():
        out = torch.full((1,) + de.BIG_OUT + (4,), 0x5A5A, dtype=torch.int16, device="cuda").view(torch.uint16)
        _, _, st = gpu.decode_packed_resized_device(*big_file, de.BIG_OUT, 4, boxes=torch.tensor([c.box], dtype=torch.int32, device="cuda"),
                                                    out=out, any_png=True, native=True)
        assert not st.any().item()
        compare(out, 0, de.big_fetch(c.box), c.crop[2:], de.BIG_OUT, c.aa, "uint16", True, 65535)
        torch.cuda.empty_cache()


def test_big_ragged_output_past_4_gib(gpu, big_file):
    """the same file decoded natively to RGBA uint16: one file's output of 4.4 GB; sampled rows, the last one included"""
    import torch
    out, oo, info, st = gpu.decode_packed_ragged_device(*big_file, 4, dtype=torch.uint16, any_png=True, native=True)
    assert not st.any().item()
    v = gpu.ragged_views(out, oo, info, st, 4)[0]
    rows = de.sample_rows(de.BIG_H, 6, 7)
    got = v.view(torch.int16)[torch.as_tensor(rows, device="cuda")].cpu().numpy().view(np.uint16).astype(np.int64)
    want = np.stack([de.big_fetch((int(r), 0))(0, 1, 0, de.BIG_W)[0] for r in rows])
    assert np.array_equal(got, want)
    del out, v
    torch.cuda.empty_cache()


def test_batch_past_4_gib(gpu):
    """9 files upscaled to 8192 x 8192 RGBA uint16: 512 MiB each, the last one placed past 4 GiB of the output"""
    import torch
    need_free(de.batch_bytes() / 1e9 + 0.5)
    srcs = [source(11 + k, 13 + 2 * k, 4, True, 40 + k) for k in range(de.BATCH_N)]
    out = resize(gpu, [p for p, _ in srcs], 4, de.BATCH_OUT, "uint16", True, True)
    rows = de.sample_rows(de.BATCH_OUT[0], 4, 8)
    for f in (0, de.BATCH_N - 1):
        px = srcs[f][1]
        compare(out, f, de.array_fetch(px), px.shape[:2], de.BATCH_OUT, True, "uint16", True, int(px.max()), rows=rows)
    del out
    torch.cuda.empty_cache()


# ---- 2. native ragged decode at its tiling edges -----------------------------------------------------------------------------
SCALE, BIAS = [0.5, -2.0, 0.125, 3.0], [1.0, 0.25, -7.0, 0.5]


def expected(m16, depth, dtype, chans):
    if dtype in ("uint8", "uint16"):
        return native_out(m16, depth, dtype)
    import torch
    x = m16.astype(np.float32) / np.float32(257.0) if depth == 16 else (m16 >> 8).astype(np.float32)
    return (torch.from_numpy(x) * torch.tensor(SCALE[:chans]) + torch.tensor(BIAS[:chans])).to(getattr(torch, dtype))


def ragged(gpu, files, d, dtype):
    import torch
    data, offsets, sizes = packed(files)
    kw = dict(scale=SCALE[:d or 4], bias=BIAS[:d or 4]) if dtype.startswith(("float", "bfloat")) else {}
    out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=getattr(torch, dtype), any_png=True,
                                                        all_formats=True, native=True, **kw)
    assert not st.any().item(), st.cpu().numpy()
    return gpu.ragged_views(out, oo, info, st, d)


def same(got, want):
    import torch
    if isinstance(want, torch.Tensor):
        return torch.equal(got.cpu(), want)
    return np.array_equal(as_np(got), want)


@pytest.fixture(scope="module")
def fpng_files(oracle):
    out = []
    for w, h, c, stored in de.fpng_shapes():
        img = de.fpng_image(w, h, c, stored, w + h)
        out.append((oracle.encode(img, w, h, c, 0), img))
    return out


@pytest.mark.parametrize("dtype", ["uint8", "uint16", "float16", "bfloat16"])
def test_fpng_ragged_cta_edges(gpu, fpng_files, dtype):
    """fpng files 511 .. 2049 wide (one to five unfilter CTAs) and 1 .. 17 high (around the 8 rows loaded ahead), stored and
    Huffman coded, at desired 0 .. 4"""
    for d in (0, 1, 2, 3, 4):
        views = ragged(gpu, [f for f, _ in fpng_files], d, dtype)
        for k, (_, img) in enumerate(fpng_files):
            c = d or img.shape[2]
            assert same(views[k], expected(fpng_native16(img, d), 8, dtype, c)), (d, dtype, img.shape)


@pytest.fixture(scope="module")
def general_files():
    rs = np.random.RandomState(61)
    return [(pf.case(rs, w, h, ct, 8, seed=k), ct) for k, (w, h, ct) in enumerate(de.general_shapes())]


@pytest.mark.parametrize("d,dtype", [(0, "uint8"), (0, "uint16"), (1, "uint16"), (1, "float16"), (2, "uint16"), (2, "float16")])
def test_general_bands_in_one_call(gpu, general_files, d, dtype):
    """8-bit gray, gray+alpha, RGB and RGBA files with random filters, 31 .. 97 rows (one to four 32-row bands) in one call"""
    views = ragged(gpu, [c[0][0] for c in general_files], d, dtype)
    for k, ((png, s, plte, trns), ct) in enumerate(general_files):
        m = native16(s, ct, 8, d)
        assert same(views[k], expected(m, 8, dtype, m.shape[2])), (d, dtype, s.shape, ct)


@pytest.fixture(scope="module")
def ext_files():
    rs = np.random.RandomState(62)
    return [(pf.case(rs, w, h, ct, depth, il, t, seed=k), ct, depth) for k, (ct, depth, il, t, w, h) in enumerate(de.ext_specs())]


@pytest.mark.parametrize("dtype", ["uint8", "uint16"])
@pytest.mark.parametrize("d", [0, 1, 2])
def test_ext_bands(gpu, ext_files, d, dtype):
    """Adam7 files whose every pass has two bands or more, palette and gray 1/2/4-bit at widths 8k - 1, 8k, 8k + 1, and 16-bit
    files with a color key"""
    views = ragged(gpu, [c[0][0] for c in ext_files], d, dtype)
    for k, ((png, s, plte, trns), ct, depth) in enumerate(ext_files):
        m = native16(s, ct, depth, d, plte, trns)
        assert same(views[k], expected(m, depth, dtype, m.shape[2])), (d, dtype, s.shape, ct, depth)
