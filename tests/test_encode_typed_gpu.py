"""GPU tests of the typed encode (fpngb_encode_*_typed): float32 / float16 / bfloat16 input with a per-channel scale and bias,
rounded to 8 bits by the conversion pre-pass.  Every file must be byte-identical to what the uint8 encode writes for
torch.nan_to_num(x.float() * s + b, nan=0).round().clamp(0, 255).to(torch.uint8), for every layout, width and flag; rejected
calls must launch nothing and write nothing."""
import ctypes as C

import numpy as np
import pytest

import imagegen
from test_encode_typed_cpu import CLIP, IMAGENET, PM1, UNIT, round_trip
from test_trained_tables_cpu import load_tables

pytestmark = pytest.mark.gpu

DTYPES = ("float32", "float16", "bfloat16")
WIDTHS = (1, 2, 3, 5, 67, 687, 1920)
LAYOUTS = ("nhwc", "nchw_padded", "crop", "hcw", "broadcast")
FLAGS = (0, 1, 2)
ERR_INVALID_ARG, ERR_ALIGNMENT = 1, 5
GUARD = 0xA5


def tdt(name):
    import torch
    return getattr(torch, name)


def quantize(x, s, b):
    """the contract, in torch on the device"""
    import torch
    s = torch.as_tensor(np.asarray(s, np.float32), device=x.device)
    b = torch.as_tensor(np.asarray(b, np.float32), device=x.device)
    return torch.nan_to_num(x.float() * s + b, nan=0.0).round().clamp(0, 255).to(torch.uint8)


def files_of(out, sizes):
    sizes = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    out = out.cpu().numpy()
    return [out[i, : sizes[i]].tobytes() for i in range(len(sizes))]


def ragged_files(out, offsets, sizes):
    """the files of an encode_ragged_device result (the bytes of a slot past its file are not written)"""
    o = offsets.cpu().numpy()
    s = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    out = out.cpu().numpy()
    return [out[o[i]:o[i] + s[i]].tobytes() for i in range(len(s))]


def float_images(n, h, w, c, dtype, seed, affine):
    """[n, h, w, c] floats on the device from imagegen pixels: ties, out-of-range values, NaN and +-inf in a fraction of the
    elements; with affine "pm1" the values are (v - 127.5) / 127.5, encoded with scale = bias = 127.5"""
    import torch
    rng = np.random.RandomState(seed)
    u8 = np.stack([imagegen.make("g1" if i % 2 == 0 else "runs", w, h, c, seed + i).reshape(h, w, c) for i in range(n)])
    v = u8.astype(np.float32) + rng.choice(np.float32([0.0, 0.5, -0.5, 0.25, 0.49999997, -0.75]), size=u8.shape)
    special = rng.rand(*u8.shape) < 0.04
    v[special] = rng.choice(np.float32([np.nan, np.inf, -np.inf, 300.0, -20.0, 1e30, -0.0, 255.5]), size=int(special.sum()))
    s, b = np.float32([1.0] * c), np.float32([0.0] * c)
    if affine == "pm1":
        v = (v - np.float32(127.5)) / np.float32(127.5)
        s, b = np.float32([127.5] * c), np.float32([127.5] * c)
    elif affine == "mixed":
        s = np.float32([1.0, 0.5, 2.0, -1.0])[:c]
        b = np.float32([0.0, 64.0, -100.0, 255.0])[:c]
    return torch.from_numpy(v).cuda().to(tdt(dtype)), s, b


def view_as(x, layout):
    """x [n, h, w, c] contiguous -> the same values in the given layout"""
    import torch
    n, h, w, c = x.shape
    if layout == "nhwc":
        return x
    if layout == "nchw_padded":                                             # plane stride h*w + 3 elements
        cs = h * w + 3
        flat = torch.full((n * c * cs + 8,), float("nan"), dtype=x.dtype, device=x.device)
        view = flat.as_strided((n, h, w, c), (c * cs, w, 1, cs), 1)
        view.copy_(x)
        return view
    if layout == "crop":
        canvas = torch.full((n, h + 2, w + 5, c), float("nan"), dtype=x.dtype, device=x.device)
        canvas[:, 1:1 + h, 3:3 + w] = x
        return canvas[:, 1:1 + h, 3:3 + w]
    if layout == "hcw":
        return x.permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)
    assert layout == "broadcast"
    return x[:1].expand(n, -1, -1, -1)


def launches(gpu, fn):
    import torch
    torch.cuda.synchronize()
    before = gpu.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return gpu.launch_count() - before, r


# ---- 1. byte identity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [3, 4])
def test_byte_identity(gpu, dtype, c):
    for k, w in enumerate(WIDTHS):
        h = 3 if w >= 687 else 5
        for affine in ("id", "pm1", "mixed"):
            x, s, b = float_images(3, h, w, c, dtype, 100 * k + c, affine)
            for layout in LAYOUTS:
                view = view_as(x, layout)
                q = quantize(view, s, b).contiguous()
                for flags in FLAGS:
                    want = files_of(*gpu.encode_batch_device(q, flags))
                    got = files_of(*gpu.encode_batch_device(view, flags, scale=s, bias=b))
                    assert got == want, (dtype, c, w, affine, layout, flags)


def test_one_scale_for_every_channel_and_defaults(gpu):
    import torch
    x, _, _ = float_images(2, 7, 33, 3, "float32", 5, "id")
    for kw, (s, b) in (({}, ([1.0] * 3, [0.0] * 3)), ({"scale": 0.5}, ([0.5] * 3, [0.0] * 3)), ({"bias": 10.0}, ([1.0] * 3, [10.0] * 3))):
        want = files_of(*gpu.encode_batch_device(quantize(x, s, b), 0))
        assert files_of(*gpu.encode_batch_device(x, 0, **kw)) == want, kw
    # entries beyond the channel count are ignored by the C call: a NaN there is accepted
    from fpng_b200._lib import PixelFormat, lib
    fmt = PixelFormat()
    fmt.dtype = 1
    fmt.scale[:] = [1.0, 1.0, 1.0, float("nan")]
    fmt.bias[:] = [0.0, 0.0, 0.0, float("inf")]
    out =torch.empty((2, (gpu.max_encoded_size(33, 7, 3) + 15) // 16 * 16), dtype=torch.uint8, device="cuda")
    sizes = torch.empty(2, dtype=torch.int32, device="cuda")
    assert lib().fpngb_encode_batch_device_typed(x.data_ptr(), 7 * 33 * 12, 33 * 12, 12, 4, 2, 33, 7, 3, C.byref(fmt), 0,
                                                 out.data_ptr(), out.stride(0), sizes.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert files_of(out, sizes) == files_of(*gpu.encode_batch_device(quantize(x, [1.0] * 3, [0.0] * 3), 0))


# ---- 2. round trip ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_round_trip_decode_normalise_encode_denormalise(gpu, dtype):
    import torch
    from fpng_b200 import denormalize_scale_bias, normalize_scale_bias
    from test_decode_device_gpu import packed_device
    w, h, n = 256, 3, 2
    ramp = np.arange(256, dtype=np.uint8)
    imgs = np.stack([np.stack([np.roll(ramp, 7 * i + y)[:, None].repeat(3, 1) for y in range(h)]) for i in range(n)])
    imgs[1, 1] = 255 - imgs[1, 1]
    for flags in FLAGS:
        files = files_of(*gpu.encode_batch_device(torch.from_numpy(imgs).cuda(), flags))
        data, offsets, sizes = packed_device(files)
        for name, (mean, std) in (("unit", UNIT), ("pm1", PM1), ("imagenet", IMAGENET), ("clip", CLIP)):
            sn, bn = normalize_scale_bias(mean, std)
            sd, bd = denormalize_scale_bias(mean, std)
            nchw = torch.empty((n, 3, h, w), dtype=tdt(dtype), device="cuda")
            _, st = gpu.decode_packed_device(data, offsets, sizes, w, h, 3, 3, out=nchw.permute(0, 2, 3, 1), scale=sn, bias=bn)
            assert (st.cpu() == 0).all()
            x = nchw.permute(0, 2, 3, 1)
            got = files_of(*gpu.encode_batch_device(x, flags, scale=sd, bias=bd))
            assert got == files_of(*gpu.encode_batch_device(quantize(x, sd, bd).contiguous(), flags)), (name, flags)
            exact = bool((round_trip(tdt(dtype), mean, std) == torch.arange(256, dtype=torch.uint8)[:, None]).all())
            if exact:
                assert got == files, (dtype, name, flags)


# ---- 3. ragged -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_ragged_mixed_shapes_channels_layouts(gpu, dtype):
    import torch
    shapes = [(5, 1, 3), (3, 2, 4), (7, 67, 3), (2, 687, 4), (4, 1920, 3), (9, 5, 4), (1, 3, 3), (40, 200, 4)]
    layouts = ("nhwc", "nchw_padded", "crop", "hcw")
    views, qs = [], []
    for i, (h, w, c) in enumerate(shapes):
        x, _, _ = float_images(1, h, w, c, dtype, 7 + i, "pm1")
        v = view_as(x, layouts[i % len(layouts)])[0]
        views.append(v)
        qs.append(v)
    s, b = [127.5] * 4, [127.5] * 4
    qs = [quantize(v, s[:v.shape[2]], b[:v.shape[2]]).contiguous() for v in views]
    for flags in FLAGS:
        out, offs, sizes = gpu.encode_ragged_device(views, flags, scale=s, bias=b)
        ref_out, ref_offs, ref_sizes = gpu.encode_ragged_device(qs, flags)
        torch.cuda.synchronize()
        assert torch.equal(offs, ref_offs) and torch.equal(sizes, ref_sizes), flags
        assert ragged_files(out, offs, sizes) == ragged_files(ref_out, ref_offs, ref_sizes), (dtype, flags)
        dec, _, info, st = gpu.decode_packed_ragged_device(out, offs, sizes, 4)
        assert (st.cpu() == 0).all()
        for i, v in enumerate(gpu.ragged_views(dec, _, info, st, 4)):
            c = shapes[i][2]
            assert torch.equal(v[..., :c], qs[i]), (dtype, flags, i)


# ---- 4. fallbacks ----------------------------------------------------------------------------------------------------------
def test_trained_table_rule_and_fused_encoder(gpu, oracle):
    import torch
    from fpng_b200._lib import lib
    L = lib()
    t = load_tables()["4"]
    prefix = bytes.fromhex(t["prefix"])
    table_sizes = np.array(t["sizes"], np.uint8)
    w, h = 61, 24
    pal = [int(v) for v in np.argsort(table_sizes[:256], kind="stable")[:4]]
    src = np.stack([imagegen.short_runs(w, h, 4, 7 + i, pal) for i in range(4)])
    x = torch.from_numpy(src).cuda().float().add_(0.25).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    q = quantize(x, [1.0] * 4, [0.0] * 4).contiguous()
    assert torch.equal(q.cpu(), torch.from_numpy(src))

    def check(flags):
        base, want = launches(gpu, lambda: files_of(*gpu.encode_batch_device(q, flags)))
        k, got = launches(gpu, lambda: files_of(*gpu.encode_batch_device(x, flags, scale=1.0)))
        assert got == want and k == base + 1, (flags, k, base)          # one conversion launch, no copy of the converted rows
        return got

    oracle.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
    try:
        gpu.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
        got = check(0)
        for i in range(4):
            assert got[i] == oracle.encode(src[i], w, h, 4, 0), i
        # the ragged call sends these images through the uniform pipeline one at a time: same bytes as the uint8 call
        res = gpu.encode_ragged_device([x[i] for i in range(4)], 0, scale=1.0)
        ref = gpu.encode_ragged_device([q[i] for i in range(4)], 0)
        torch.cuda.synchronize()
        assert torch.equal(res[1], ref[1]) and ragged_files(*res) == ragged_files(*ref) == got
    finally:
        gpu.set_static_table(4)
        oracle.set_static_table(4)
    try:
        L.fpngb_debug_use_fused(1)
        for c in (3, 4):
            xf, s, b = float_images(3, 30, 640, c, "bfloat16", 3, "mixed")
            xv = view_as(xf, "nchw_padded")
            qf = quantize(xv, s, b).contiguous()
            for flags in (0, 1):
                base, want = launches(gpu, lambda: files_of(*gpu.encode_batch_device(qf, flags)))
                k, got = launches(gpu, lambda: files_of(*gpu.encode_batch_device(xv, flags, scale=s, bias=b)))
                assert got == want and k == base + 1, (c, flags, k, base)
    finally:
        L.fpngb_debug_use_fused(-1)


# ---- 5. rejections ---------------------------------------------------------------------------------------------------------
def test_rejections_launch_nothing_write_nothing(gpu):
    import torch
    from fpng_b200._lib import PixelFormat, lib
    L = lib()
    n, h, w, c = 2, 4, 8, 3
    x = torch.rand((n, h, w, 4), device="cuda") * 255
    cap = (gpu.max_encoded_size(w, h, c) + 15) // 16 * 16
    out = torch.full((n, cap), GUARD, dtype=torch.uint8, device="cuda")
    sizes = torch.full((n,), -1, dtype=torch.int32, device="cuda")

    def fmt_of(dtype=1, scale=(1.0,) * 4, bias=(0.0,) * 4):
        f = PixelFormat()
        f.dtype = dtype
        f.scale[:] = list(scale)
        f.bias[:] = list(bias)
        return f

    good = fmt_of()
    rgb = x[..., :3].contiguous()
    es = 4
    tight = (h * w * c * es, w * c * es, c * es, es)
    cases = [
        (ERR_INVALID_ARG, rgb.data_ptr(), tight, None),
        (ERR_INVALID_ARG, rgb.data_ptr(), tight, fmt_of(dtype=0)),
        (ERR_INVALID_ARG, rgb.data_ptr(), tight, fmt_of(dtype=4)),
        (ERR_INVALID_ARG, rgb.data_ptr(), tight, fmt_of(scale=(1.0, float("nan"), 1.0, 1.0))),
        (ERR_INVALID_ARG, rgb.data_ptr(), tight, fmt_of(bias=(0.0, 0.0, float("-inf"), 0.0))),
        (ERR_ALIGNMENT, rgb.data_ptr() + 2, tight, good),
        (ERR_ALIGNMENT, rgb.data_ptr(), (tight[0], tight[1] + 2, tight[2], tight[3]), good),
        (ERR_ALIGNMENT, rgb.data_ptr(), (tight[0] + 1, tight[1], tight[2], tight[3]), good),
        (ERR_INVALID_ARG, x.data_ptr(), (h * w * 16, w * 16, 16, 4), good),                  # RGB view of RGBA floats
    ]
    torch.cuda.synchronize()
    before = gpu.launch_count()
    for want, ptr, st, f in cases:
        rc = L.fpngb_encode_batch_device_typed(ptr, *st, n, w, h, c, C.byref(f) if f is not None else None, 0, out.data_ptr(), cap,
                                               sizes.data_ptr(), None)
        assert rc == want, (want, rc, st)
    # the ragged call: the same rules per image
    dims = np.array([[w, h, c]] * 2, np.uint32)
    ptrs = np.array([rgb.data_ptr(), rgb.data_ptr()], np.uint64)
    flat = torch.full((2 * cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    offs = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    for want, p1, strides, f in [
        (ERR_INVALID_ARG, rgb.data_ptr(), None, fmt_of(dtype=0)),
        (ERR_INVALID_ARG, rgb.data_ptr(), None, None),
        (ERR_INVALID_ARG, rgb.data_ptr(), None, fmt_of(scale=(1.0, 1.0, float("inf"), 1.0))),
        (ERR_ALIGNMENT, rgb.data_ptr() + 6, None, good),
        (ERR_ALIGNMENT, rgb.data_ptr(), np.array([[w * c * 4, c * 4, 4], [w * c * 4 + 3, c * 4, 4]], np.uint64), good),
        (ERR_INVALID_ARG, x.data_ptr(), np.array([[w * 16, 16, 4]] * 2, np.uint64), good),
    ]:
        ptrs[1] = p1
        rc = L.fpngb_encode_ragged_device_typed(2, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p),
                                                strides.ctypes.data_as(C.c_void_p) if strides is not None else None,
                                                C.byref(f) if f is not None else None, 0, flat.data_ptr(), flat.numel(),
                                                offs.data_ptr(), sizes.data_ptr(), None)
        assert rc == want, (want, rc)
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out == GUARD).all() and (flat == GUARD).all() and (sizes == -1).all() and (offs == -1).all()


# ---- 6. addressing and streams ---------------------------------------------------------------------------------------------
def test_input_beyond_4gib(gpu):
    import torch
    n, h, w, c = 2, 6, 64, 3
    x, s, b = float_images(n, h, w, c, "float32", 17, "mixed")
    img = h * w * c
    istride = (1 << 30) + 96                                              # elements: image 1 starts 4 GiB + 384 bytes in
    buf = torch.full((istride + img + 64,), float("nan"), dtype=torch.float32, device="cuda")
    big = buf.as_strided((n, h, w, c), (istride, w * c, c, 1))
    big.copy_(x)
    want = files_of(*gpu.encode_batch_device(quantize(x, s, b), 0))
    assert files_of(*gpu.encode_batch_device(big, 0, scale=s, bias=b)) == want
    # a row pitch past 2^32 bytes (the uint8 calls stop at 2^32)
    rows = buf.as_strided((1, 2, w, c), (0, (1 << 30) + 8, c, 1))
    rows.copy_(x[:1, :2])
    want = files_of(*gpu.encode_batch_device(quantize(x[:1, :2], s, b), 0))
    assert files_of(*gpu.encode_batch_device(rows, 0, scale=s, bias=b)) == want
    res = gpu.encode_ragged_device([rows[0], big[1]], 0, scale=s, bias=b)
    ref = gpu.encode_ragged_device([quantize(rows[0], s, b).contiguous(), quantize(big[1], s, b).contiguous()], 0)
    torch.cuda.synchronize()
    assert ragged_files(*res) == ragged_files(*ref)
    del buf, big, rows
    torch.cuda.empty_cache()


def test_streams_overlap_and_profile_slot(gpu):
    import torch
    from fpng_b200._lib import lib
    L = lib()
    xa, sa, ba = float_images(8, 256, 512, 3, "bfloat16", 1, "pm1")
    xb, sb, bb = float_images(6, 200, 300, 4, "float32", 2, "mixed")
    u8 = torch.from_numpy(np.stack([imagegen.make("g1", 400, 150, 3, 30 + i).reshape(150, 400, 3) for i in range(8)])).cuda()
    va, vb = view_as(xa, "nchw_padded"), view_as(xb, "crop")
    want_a = files_of(*gpu.encode_batch_device(quantize(va, sa, ba).contiguous(), 0))
    want_b = files_of(*gpu.encode_batch_device(quantize(vb, sb, bb).contiguous(), 1))
    want_u = files_of(*gpu.encode_batch_device(u8, 0))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    for _ in range(3):
        res = []
        for st, fn in zip(streams, (lambda: gpu.encode_batch_device(va, 0, scale=sa, bias=ba),
                                    lambda: gpu.encode_batch_device(vb, 1, scale=sb, bias=bb),
                                    lambda: gpu.encode_batch_device(u8, 0))):
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                res.append(fn())
        torch.cuda.synchronize()
        assert files_of(*res[0]) == want_a and files_of(*res[1]) == want_b and files_of(*res[2]) == want_u
    ms = (C.c_float * 10)()
    L.fpngb_profile_read(ms, 10)                                           # drop earlier calls
    L.fpngb_profile_enable(1)
    try:
        gpu.encode_batch_device(va, 0, scale=sa, bias=ba)
        assert L.fpngb_profile_read(ms, 10) == 1
        assert ms[9] > 0 and ms[6] > 0, list(ms)
        gpu.encode_batch_device(u8, 0)
        ms9 = (C.c_float * 9)()
        assert L.fpngb_profile_read(ms9, 9) == 1 and ms9[6] > 0
        gpu.encode_batch_device(u8, 0)
        assert L.fpngb_profile_read(ms, 10) == 1 and ms[9] == 0            # a uint8 call runs no conversion
    finally:
        L.fpngb_profile_enable(0)
