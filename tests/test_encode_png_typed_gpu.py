"""GPU tests of the typed PNG encode (encode_png_device with float images, fpngb_encode_png_ragged_device_typed): float32 / float16
/ bfloat16 input at 1 to 4 channels written as 8- or 16-bit samples.  Every file must be byte-identical to what the untyped call
writes for torch.nan_to_num(x.float() * s + b, nan=0).round().clamp(0, 2**depth - 1) as uint8 / uint16, and so to the oracles;
rejected calls must launch nothing and write nothing."""
import ctypes as C
import threading

import numpy as np
import pytest

import pngenc_workloads as pw
from test_encode_png_gpu import files
from test_trained_tables_cpu import load_tables

pytestmark = pytest.mark.gpu

DTYPES = ("float32", "float16", "bfloat16")
INVALID_ARG, TOO_SMALL, ALIGNMENT = 1, 2, 5
GUARD = 0xA5


@pytest.fixture(scope="module")
def png_oracle():
    from oracle.pngenc_oracle import PngEncodeOracle
    return PngEncodeOracle()


def tdt(name):
    import torch
    return getattr(torch, name)


def quantize(x, s, b, depth):
    """the contract, in torch on x's device"""
    import torch
    s = torch.as_tensor(np.asarray(s, np.float32), device=x.device)
    b = torch.as_tensor(np.asarray(b, np.float32), device=x.device)
    q = torch.nan_to_num(x.float() * s + b, nan=0.0).round().clamp(0, (1 << depth) - 1)
    return q.to(torch.uint8 if depth == 8 else torch.uint16)


def float_image(h, w, c, dtype, depth, seed):
    """[h, w, c] floats on the device roughly in [-0.1, 1.1] with NaN, +-inf, -0, 1e30 and out-of-range values in a fraction of
    the elements, for scale ~ 2**depth - 1"""
    import torch
    rng = np.random.default_rng(seed)
    v = rng.uniform(-0.1, 1.1, (h, w, c)).astype(np.float32)
    special = rng.random((h, w, c)) < 0.05
    v[special] = rng.choice(np.float32([np.nan, np.inf, -np.inf, -0.0, 1e30, -1e30, 2.0, -1.0]), size=int(special.sum()))
    return torch.from_numpy(v).cuda().to(tdt(dtype))


def tie_image(h, w, c, dtype, depth, seed):
    """[h, w, c] exact ties k + 0.5 of the output grid (k small enough for the dtype to hold them), for scale 1 and bias 0"""
    import torch
    top = {"float32": (1 << depth) - 1, "float16": 1023, "bfloat16": 127}[dtype]
    rng = np.random.default_rng(seed)
    v = rng.integers(0, top + 1, (h, w, c)).astype(np.float32) + np.float32(0.5)
    v[0, 0, 0] = (1 << depth) - 0.5 if dtype == "float32" else v[0, 0, 0]
    return torch.from_numpy(v).cuda().to(tdt(dtype))


def launches(gpu, fn):
    import torch
    torch.cuda.synchronize()
    before = gpu.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return gpu.launch_count() - before, r


def host(q):
    return q.contiguous().cpu().numpy()


# ---- 1. every dtype, channel count, depth and flag --------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, 1, 2])
@pytest.mark.parametrize("depth", [8, 16])
@pytest.mark.parametrize("c", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_format(gpu, png_oracle, dtype, c, depth, flags):
    M = float((1 << depth) - 1)
    scale = np.float32([M, 0.5 * M, -M, 1.25 * M])[:c]
    bias = np.float32([0.0, 0.25 * M, M, -0.1 * M])[:c]
    shapes = [(3, 1), (5, 17), (9, 67), (2, 260)]
    xs = [float_image(h, w, c, dtype, depth, 100 * c + k) for k, (h, w) in enumerate(shapes)]
    for x, s, b in ((xs, scale, bias), ([tie_image(7, 45, c, dtype, depth, c)], None, None)):
        sq, bq = (s if s is not None else [1.0] * c), (b if b is not None else [0.0] * c)
        qs = [quantize(t, sq, bq, depth).contiguous() for t in x]
        got = files(*gpu.encode_png_device(x, flags, scale=s, bias=b, depth=depth))
        assert got == files(*gpu.encode_png_device(qs, flags)), (dtype, c, depth, flags)
        for k, q in enumerate(qs):
            if depth == 8 and c >= 3:
                continue
            assert got[k] == png_oracle.png_encode(host(q), flags), (dtype, c, depth, flags, k)
        if depth == 8 and c >= 3:
            assert got == files(*gpu.encode_ragged_device(x, flags, scale=s, bias=b))


# ---- 2. layouts, read in place ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_layouts(gpu, png_oracle, dtype):
    import torch
    es = torch.empty((), dtype=tdt(dtype)).element_size()
    views, depths = [], []
    for c in (1, 2, 3, 4):
        depth = 16 if c % 2 else 8
        canvas = float_image(21, 37, c, dtype, depth, 7 + c)
        views.append(canvas[2:19, 3:30]); depths.append(depth)                            # crop: row pitch of 37 pixels
        chw = canvas.permute(2, 0, 1).contiguous()
        views.append(chw.permute(1, 2, 0)); depths.append(16)                             # CHW planes
        views.append(canvas[:1].expand(9, -1, -1)); depths.append(8)                      # row stride 0
        if es == 2:                                                                         # 2-byte aligned, not 4
            flat = torch.empty((21 * 37 * c + 1,), dtype=tdt(dtype), device="cuda")
            odd = flat[1:].view(21, 37, c)
            odd.copy_(canvas)
            assert odd.data_ptr() % 4 == 2
            views.append(odd); depths.append(16)
    assert views[1].stride()[1] == 1 and views[2].stride()[0] == 0
    s = [1000.0, 200.0, 60000.0, 255.0]
    got = files(*gpu.encode_png_device(views, 0, scale=s, depth=depths))
    qs = [quantize(v, s[:v.shape[2]], [0.0] * v.shape[2], d).contiguous() for v, d in zip(views, depths)]
    assert got == files(*gpu.encode_png_device(qs, 0))
    for k, (q, d) in enumerate(zip(qs, depths)):
        if not (d == 8 and q.shape[2] >= 3):
            assert got[k] == png_oracle.png_encode(host(q), 0), k


def test_row_stride_past_4gib(gpu):
    """a float32 view whose row stride passes 4 GiB: the typed call reads it (64-bit input addressing); the untyped call, whose
    row kernels take a 32-bit pitch, refuses the same byte layout"""
    import torch
    w, c = 50, 2
    rs = (1 << 30) + 8                                                    # elements: 4 GiB + 32 bytes
    buf = torch.zeros((rs + w * c + 16,), dtype=torch.float32, device="cuda")
    rows = buf.as_strided((2, w, c), (rs, c, 1))
    src = float_image(2, w, c, "float32", 16, 5)
    rows.copy_(src)
    want = files(*gpu.encode_png_device([quantize(src, [65535.0], [0.0], 16).contiguous()], 0))
    assert files(*gpu.encode_png_device([rows], 0, scale=65535.0, depth=16)) == want
    as_u16 = buf.view(torch.uint16).as_strided((2, w, c), (2 * rs, c, 1))
    from fpng_b200._lib import FpngB200Error
    with pytest.raises(FpngB200Error):
        gpu.encode_png_device([as_u16], 0)
    del buf, rows, as_u16
    torch.cuda.empty_cache()


# ---- 3. one call mixing depths, channel counts and fpng images -------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, 1, 2])
def test_mixed_call(gpu, png_oracle, flags):
    import torch
    images, depths = [], []
    for k in range(16):
        c, depth = 1 + k % 4, (8, 16)[(k // 4) % 2]
        h, w = 3 + (k * 7) % 11, 1 + (k * 13) % 40
        images.append(float_image(h, w, c, "bfloat16", depth, 300 + k)); depths.append(depth)
    s, b = [250.0, 60000.0, 255.0, 30000.0], [2.0, 0.0, 1.0, 4.0]
    out, offsets, sizes = gpu.encode_png_device(images, flags, scale=s, bias=b, depth=depths)
    shapes = [(t.shape[0], t.shape[1], t.shape[2], d) for t, d in zip(images, depths)]
    torch.cuda.synchronize()
    assert offsets.cpu().numpy().tolist() == gpu.png_slot_offsets(shapes).tolist()
    got = files(out, offsets, sizes)
    qs = [quantize(t, s[:t.shape[2]], b[:t.shape[2]], d).contiguous() for t, d in zip(images, depths)]
    assert got == files(*gpu.encode_png_device(qs, flags))
    for k, (q, d) in enumerate(zip(qs, depths)):
        if not (d == 8 and q.shape[2] >= 3):
            assert got[k] == png_oracle.png_encode(host(q), flags), k


def test_trained_table_typed_call(gpu, oracle):
    """RGBA 1-pass under a table whose one-pixel-match rule is live: the typed call writes the untyped call's files with one
    launch more, its conversion kernel; both stay in the ragged pipeline"""
    import torch
    t = load_tables()["4"]
    prefix = bytes.fromhex(t["prefix"])
    x = [float_image(24, 61, 4, "float16", 8, 40 + i) for i in range(3)] + [float_image(9, 20, 1, "float16", 16, 50)]
    depths = [8, 8, 8, 16]
    qs = [quantize(v, [255.0], [0.0], d).contiguous() for v, d in zip(x, depths)]
    oracle.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
    try:
        gpu.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
        base, want = launches(gpu, lambda: files(*gpu.encode_png_device(qs, 0)))
        k, got = launches(gpu, lambda: files(*gpu.encode_png_device(x, 0, scale=255.0, depth=depths)))
        assert got == want and k == base + 1
        for i in range(3):
            q = host(qs[i])
            assert got[i] == oracle.encode(q, 61, 24, 4, 0), i
    finally:
        gpu.set_static_table(4)
        oracle.set_static_table(4)
    torch.cuda.synchronize()


# ---- 4. round trip through the native float decode -------------------------------------------------------------------------
def test_round_trip_native_decode(gpu):
    """encode with the uint call, decode natively into float32 (8-bit files at scale 1, 16-bit files at 0.257: metres from
    millimetres), re-encode with the inverse scale: the same files, byte for byte"""
    import torch
    corpus = [img for _, img in pw.corpus()]
    groups = {8: [i for i in corpus if i.dtype == np.uint8] + pw.workload("E1", 4) + pw.workload("E3", 3),
              16: [i for i in corpus if i.dtype == np.uint16] + pw.workload("E2", 4) + pw.workload("E4", 3)}
    for depth, k, inv in ((8, 1.0, 1.0), (16, 0.257, 1000.0)):
        imgs = [torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in groups[depth]]
        out, offsets, sizes = gpu.encode_png_device(imgs)
        fx, fofs, info, status = gpu.decode_packed_ragged_device(out, offsets[:-1].contiguous(), sizes, 0, any_png=True,
                                                                 all_formats=True, native=True, dtype=torch.float32, scale=k)
        views = gpu.ragged_views(fx, fofs, info, status, 0)
        assert all(v is not None for v in views)
        again = gpu.encode_png_device(views, 0, scale=inv, depth=depth)
        torch.cuda.synchronize()
        assert torch.equal(again[1], offsets)
        assert files(*again) == files(out, offsets, sizes), depth


# ---- 5. rejections ----------------------------------------------------------------------------------------------------------
def test_rejections_enqueue_nothing(gpu):
    import torch
    from fpng_b200._lib import PixelFormat, lib
    L = lib()
    x = torch.rand((4, 5, 4), device="cuda")
    out = torch.full((1 << 16,), GUARD, dtype=torch.uint8, device="cuda")
    offs = torch.full((3,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((2,), -7, dtype=torch.int32, device="cuda")

    def fmt_of(dtype=1, scale=(1.0,) * 4, bias=(0.0,) * 4):
        f = PixelFormat()
        f.dtype = dtype
        f.scale[:] = list(scale)
        f.bias[:] = list(bias)
        return f

    good = fmt_of()

    def call(dims, fmt=good, flags=0, n=None, ptr=None, strides=None, cap=1 << 16, out_ptr=None):
        dims = np.array(dims, np.uint32).reshape(-1, 4)
        n = len(dims) if n is None else n
        ptrs = np.array([x.data_ptr() if ptr is None else ptr] * len(dims), np.uint64)
        st = None if strides is None else np.array(strides, np.uint64).reshape(-1, 3).ctypes.data_as(C.c_void_p)
        return L.fpngb_encode_png_ragged_device_typed(n, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), st,
                                                      None if fmt is None else C.byref(fmt), flags,
                                                      out.data_ptr() if out_ptr is None else out_ptr, cap, offs.data_ptr(),
                                                      sizes.data_ptr(), None)

    torch.cuda.synchronize()
    before = gpu.launch_count()
    assert call([5, 4, 1, 16], fmt=None) == INVALID_ARG
    for dt in (0, 4, 5):
        assert call([5, 4, 1, 16], fmt=fmt_of(dtype=dt)) == INVALID_ARG, dt
    assert call([[5, 4, 1, 16], [5, 4, 2, 8]], fmt=fmt_of(scale=(1.0, float("nan"), 1.0, 1.0))) == INVALID_ARG
    assert call([5, 4, 3, 16], fmt=fmt_of(bias=(0.0, 0.0, float("inf"), 0.0))) == INVALID_ARG
    assert call([5, 4, 1, 16], ptr=x.data_ptr() + 2) == ALIGNMENT                 # float32 at a 2-byte address
    assert call([5, 4, 2, 16], strides=[5 * 16 + 2, 16, 4]) == ALIGNMENT          # row stride not a multiple of 4
    assert call([5, 4, 2, 8], fmt=fmt_of(dtype=2), ptr=x.data_ptr() + 1) == ALIGNMENT
    # the untyped call's rejections
    assert call([5, 4, 1, 12]) == INVALID_ARG
    assert call([5, 4, 0, 16]) == INVALID_ARG
    assert call([5, 4, 5, 16]) == INVALID_ARG
    assert call([5, 4, 1, 16], flags=4) == INVALID_ARG
    assert call([5, 4, 1, 16], n=0) == INVALID_ARG
    assert call([5, 4, 1, 16], ptr=0) == INVALID_ARG
    assert call([1 << 24, 40, 4, 16]) == INVALID_ARG
    assert call([5, 0, 1, 16]) == INVALID_ARG
    assert call([5, 4, 1, 16], cap=16) == TOO_SMALL
    assert call([5, 4, 1, 16], out_ptr=out.data_ptr() + 8) == ALIGNMENT
    assert call([5, 4, 2, 8], strides=[5 * 16, 12, 4]) == INVALID_ARG             # neither interleaved nor planar
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out == GUARD).all().item() and (offs == -7).all().item() and (sizes == -7).all().item()
    # a NaN at an index no image uses is ignored
    assert call([5, 4, 1, 16], fmt=fmt_of(scale=(65535.0, float("nan"), float("inf"), 1.0), bias=(0.0, float("nan"), 0, 0))) == 0
    torch.cuda.synchronize()
    got = out[:int(sizes[0].item())].cpu().numpy().tobytes()
    tight = x.reshape(-1)[:20].view(4, 5, 1)                                # NULL strides: tight rows of one channel
    want = files(*gpu.encode_png_device([quantize(tight, [65535.0], [0.0], 16).contiguous()], 0))[0]
    assert got == want


# ---- 6. launches, profiling, streams ----------------------------------------------------------------------------------------
def test_launch_count_and_profile_slot(gpu):
    import torch
    from fpng_b200._lib import lib
    L = lib()
    x = [float_image(40, 70, 1 + k % 4, "float32", (8, 16)[k % 2], 60 + k) for k in range(8)]
    x.append(float_image(30, 64, 3, "float32", 8, 70))                      # an fpng file in the same call
    depths = [(8, 16)[k % 2] for k in range(8)] + [8]
    qs = [quantize(t, [255.0], [0.0], d).contiguous() for t, d in zip(x, depths)]
    for flags in (0, 1, 2):
        base, want = launches(gpu, lambda: files(*gpu.encode_png_device(qs, flags)))
        k, got = launches(gpu, lambda: files(*gpu.encode_png_device(x, flags, scale=255.0, depth=depths)))
        assert got == want and k == base + 1, (flags, k, base)
    ms = (C.c_float * 10)()
    L.fpngb_profile_read(ms, 10)                                           # drop earlier calls
    L.fpngb_profile_enable(1)
    try:
        gpu.encode_png_device(x[:8], 0, scale=255.0, depth=depths[:8])
        assert L.fpngb_profile_read(ms, 10) == 1
        assert ms[9] > 0 and ms[6] > 0, list(ms)
        gpu.encode_png_device(x, 0, scale=255.0, depth=depths)
        assert L.fpngb_profile_read(ms, 10) == 1 and ms[9] > 0
        gpu.encode_png_device(qs, 0)
        assert L.fpngb_profile_read(ms, 10) == 1 and ms[9] == 0            # a uint call runs no conversion
    finally:
        L.fpngb_profile_enable(0)
    torch.cuda.synchronize()


def test_thousands_of_files_on_two_streams(gpu, png_oracle, oracle):
    import torch
    rng = np.random.default_rng(12)
    lists = []
    for s in range(2):
        imgs, depths = [], []
        for k in range(1500):
            c, depth = 1 + (k + s) % 4, (8, 16)[(k // 4 + s) % 2]
            h, w = int(rng.integers(1, 20)), int(rng.integers(1, 36))
            imgs.append(float_image(h, w, c, ("float32", "float16", "bfloat16")[s], depth, 10000 * s + k)); depths.append(depth)
        lists.append((imgs, depths))
    scales = [(255.0, 65535.0, 1.0, 30000.0), (65535.0, 255.0, 1000.0, 2.0)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    torch.cuda.synchronize()
    results = [None, None]

    def run(s):
        with torch.cuda.stream(streams[s]):
            results[s] = gpu.encode_png_device(lists[s][0], 0, scale=scales[s], depth=lists[s][1])

    th = [threading.Thread(target=run, args=(s,)) for s in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    for s in range(2):
        got = files(*results[s])
        for k, (img, d) in enumerate(zip(*lists[s])):
            c = img.shape[2]
            q = host(quantize(img, scales[s][:c], [0.0] * c, d))
            want = oracle.encode(q, q.shape[1], q.shape[0], c, 0) if d == 8 and c >= 3 else png_oracle.png_encode(q, 0)
            assert got[k] == want, (s, k, img.shape, d)
