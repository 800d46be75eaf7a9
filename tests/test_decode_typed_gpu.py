"""GPU tests of the typed decode (fpngb_decode_*_typed): float32 / float16 / bfloat16 output with a per-channel scale and bias,
converted in the unfilter pass.  Every element must have the bit pattern of torch.from_numpy(u8.astype(np.float32) * scale +
bias).to(dtype), u8 being the uint8 call's pixels for the same files; statuses must be the uint8 call's, and every element the
call does not own (gaps of strided views, ragged padding, failed files) must keep its sentinel bits."""
import ctypes as C

import numpy as np
import pytest

import imagegen
from test_decode_device_gpu import packed_device

pytestmark = pytest.mark.gpu

DTYPES = ("float32", "float16", "bfloat16")
WIDTHS = (1, 2, 3, 5, 67, 687)
SENTINEL = {4: 0x7F8A5A5A, 2: 0x7E5A}           # NaN payloads the decode never produces (scale and bias are finite)
ERR_INVALID_ARG, ERR_ALIGNMENT = 1, 5


def tdt(name):
    import torch
    return getattr(torch, name)


def ints(t):
    import torch
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def filled(shape, dtype):
    import torch
    t = torch.empty(shape, dtype=tdt(dtype), device="cuda")
    ints(t).fill_(SENTINEL[t.element_size()])
    return t


def scale_bias(d, kind):
    from fpng_b200 import normalize_scale_bias
    if kind == "imagenet":
        s, b = normalize_scale_bias((0.485, 0.456, 0.406, 0.5), (0.229, 0.224, 0.225, 0.25)[:4])
    else:                                                                   # float16: 255 * 1000 and -255 * 1000 overflow to +-inf
        s, b = np.array([1000.0, 1.0, -1000.0, 300.0], np.float32), np.array([-3.5, 0.25, 7.0, -65504.0], np.float32)
    return s[:d], b[:d]


def expect(u8, s, b, dtype):
    """the contract: two rounded fp32 operations, then torch's conversion"""
    import torch
    return torch.from_numpy(u8.astype(np.float32) * s + b).to(tdt(dtype)).cuda()


def corpus(gpu, w, h, c):
    """files of w x h x c: three images under the three encode modes, and one that fails (NOT_FPNG)"""
    import torch
    imgs = np.stack([imagegen.make(k, w, h, c, 40 + i) for i, k in enumerate(("g1", "runs", "g2"))])
    files = []
    for flags in (0, 1, 2):
        out, sizes = gpu.encode_batch_device(torch.from_numpy(imgs).cuda(), flags)
        sz = sizes.cpu().numpy()
        files += [out[i, :sz[i]].cpu().numpy().tobytes() for i in range(len(imgs))]
    bad = bytearray(files[0]); bad[58] ^= 0x01                              # zlib header: NOT_FPNG
    return files + [bytes(bad)]


def windows(n, h, w, d, dtype):
    """(buffer, [n, h, w, d] view into it) for tight NHWC, NCHW planes with padding, a padded-pitch crop and HCW"""
    buf = filled((n * h * w * d + 8,), dtype)
    yield "nhwc", buf, buf[:n * h * w * d].view(n, h, w, d)
    planes = filled((n, d + 1, h + 1, w + 2), dtype)
    yield "nchw", planes, planes[:, :d, :h, 1:1 + w].permute(0, 2, 3, 1)
    hwc = filled((n, h + 2, w + 3, d), dtype)
    yield "crop", hwc, hwc[:, 1:1 + h, 2:2 + w, :]
    hcw = filled((n, h, d, w + 1), dtype)
    yield "hcw", hcw, hcw[..., 1:].permute(0, 1, 3, 2)


def check_view(buf, guard, view, refs, what):
    """view[i] == refs[i] bit for bit (None: the file failed and keeps the sentinel), every other element of buf the sentinel"""
    exp = guard.clone()
    ev = exp.as_strided(view.shape, view.stride(), view.storage_offset())
    for i, r in enumerate(refs):
        if r is not None:
            ev[i].copy_(r)
    assert bool((ints(buf) == ints(exp)).all()), what


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [3, 4])
@pytest.mark.parametrize("d", [3, 4])
def test_typed_uniform_calls_bit_exact(gpu, dtype, c, d):
    import torch
    h = 5
    for w in WIDTHS:
        files = corpus(gpu, w, h, c)
        n = len(files)
        t, _, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, device="cuda")
        other = bytes(corpus(gpu, w + 1, h, c)[0])                          # another shape: FPNGB_DECODE_SHAPE_MISMATCH in the packed call
        data, offsets, psizes = packed_device(files + [other])
        mfs = max(len(f) for f in files + [other])
        u8, st8 = gpu.decode_packed_device(data, offsets, psizes, w, h, c, d, max_file_size=mfs)
        st8 = st8.cpu().numpy()
        assert st8[-2] == 1 and st8[-1] == 100 and not st8[:-2].any(), st8
        u8 = u8.cpu().numpy()
        for kind in ("imagenet",) + (("overflow",) if dtype == "float16" else ()):
            s, b = scale_bias(d, kind)
            refs = [expect(u8[i], s, b, dtype) if st8[i] == 0 else None for i in range(n + 1)]
            if kind == "overflow":
                assert bool(torch.isinf(torch.stack([r for r in refs if r is not None]).float()).any())
            for name, buf, view in windows(n + 1, h, w, d, dtype):
                guard = buf.clone()
                _, st = gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d, out=view[:n], scale=s, bias=b)
                assert np.array_equal(st.cpu().numpy(), st8[:n]), (name, w)
                check_view(buf, guard, view[:n], refs[:n], ("batch", name, w, kind))
                buf.copy_(guard)
                _, st = gpu.decode_packed_device(data, offsets, psizes, w, h, c, d, max_file_size=mfs, out=view, scale=s, bias=b)
                assert np.array_equal(st.cpu().numpy(), st8), (name, w)
                check_view(buf, guard, view, refs, ("packed", name, w, kind))


def test_typed_default_scale_bias_and_dtype_argument(gpu):
    import torch
    w, h, c = 67, 4, 3
    files = corpus(gpu, w, h, c)[:3]
    data, offsets, sizes = packed_device(files)
    u8, _ = gpu.decode_packed_device(data, offsets, sizes, w, h, c, 3)
    for dtype in DTYPES:
        out, st = gpu.decode_packed_device(data, offsets, sizes, w, h, c, 3, dtype=tdt(dtype))
        assert out.dtype == tdt(dtype) and out.is_contiguous() and int(st.abs().sum()) == 0
        assert bool((ints(out) == ints(u8.to(tdt(dtype)))).all())
    with pytest.raises(ValueError):
        gpu.decode_packed_device(data, offsets, sizes, w, h, c, 3, scale=[1.0, 1.0, 1.0])
    with pytest.raises(ValueError):
        gpu.decode_packed_device(data, offsets, sizes, w, h, c, 3, out=torch.empty((3, h, w, 3), dtype=torch.uint8, device="cuda"),
                                 bias=0.5)


# ---- ragged --------------------------------------------------------------------------------------------------------------
def ragged_corpus(gpu):
    files = []
    for (w, h, c) in ((5, 3, 3), (687, 4, 4), (1, 7, 3), (67, 2, 4), (2, 9, 3), (3, 1, 4)):
        files += corpus(gpu, w, h, c)[:2]
    bad = bytearray(files[2]); bad[58] ^= 0x01
    return files + [bytes(bad)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [3, 4])
def test_typed_ragged_bit_exact_and_untouched(gpu, dtype, d):
    import torch
    files = ragged_corpus(gpu)
    data, offsets, sizes = packed_device(files)
    s, b = scale_bias(d, "imagenet")
    u8, oo8, info8, st8 = gpu.decode_packed_ragged_device(data, offsets, sizes, d)
    views8 = gpu.ragged_views(u8, oo8, info8, st8, d)
    st8 = st8.cpu().numpy()
    assert st8[-1] == 1 and not st8[:-1].any()
    es = 4 if dtype == "float32" else 2
    # the exact total, then one that leaves the last decodable files OUT_OF_SPACE
    _, oo, _, _ = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=tdt(dtype), scale=s, bias=b)
    total = int(oo[-1])
    ends = [(int(oo[i]) + (int(info8[i, 1]) * int(info8[i, 2]) * d * es + 15) // 16 * 16) for i in range(len(files))]
    for cap in (total, ends[len(files) - 4]):
        buf = filled((cap // es + 64,), dtype)
        guard = buf.clone()
        out, oo, info, st_t = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=buf[:cap // es], scale=s, bias=b,
                                                              max_file_size=max(len(f) for f in files), max_w=687, max_h=9)
        st = st_t.cpu().numpy()
        want = st8.copy()
        if cap < total:
            want[len(files) - 3:] = 101                                     # FPNGB_DECODE_OUT_OF_SPACE
        assert np.array_equal(st, want), (cap, st)
        assert int(oo[-1]) & ((1 << 63) - 1) == total
        exp = guard.clone()
        for i, v in enumerate(gpu.ragged_views(exp[:cap // es], oo, info, st_t, d)):
            if v is not None:
                v.copy_(expect(views8[i].cpu().numpy(), s, b, dtype))
        assert bool((ints(buf) == ints(exp)).all()), cap
        views = gpu.ragged_views(out, oo, info, st_t, d)
        assert all((v is None) == (st[i] != 0) for i, v in enumerate(views))


# ---- verify mode ---------------------------------------------------------------------------------------------------------
def test_typed_verify_failures_leave_output_untouched(gpu):
    import torch
    w, h, c, d = 67, 6, 3, 3
    files = corpus(gpu, w, h, c)[:6]
    crc = bytearray(files[0]); crc[-16] ^= 0x01                             # last IDAT data byte: IDAT CRC-32 mismatch
    adl = bytearray(files[3]); adl[-17] ^= 0x01                             # a stored byte: Adler-32 mismatch (the CRC is fixed up)
    import zlib
    st0, *_rest, io, il = gpu.get_info_ex(bytes(adl))
    body = bytes(adl[io + 4:io + 8 + il])
    adl[io + 8 + il:io + 12 + il] = (zlib.crc32(body) & 0xFFFFFFFF).to_bytes(4, "big")
    files = files + [bytes(crc), bytes(adl)]
    data, offsets, sizes = packed_device(files)
    s, b = scale_bias(d, "imagenet")
    gpu.set_decode_verify(True)
    try:
        u8, st8 = gpu.decode_packed_device(data, offsets, sizes, w, h, c, d)
        st8 = st8.cpu().numpy()
        assert st8[-2] == 4 and st8[-1] in (102, 1), st8
        u8 = u8.cpu().numpy()
        for dtype in DTYPES:
            out = filled((len(files), d, h, w), dtype)
            guard = out.clone()
            _, st = gpu.decode_packed_device(data, offsets, sizes, w, h, c, d, out=out.permute(0, 2, 3, 1), scale=s, bias=b)
            assert np.array_equal(st.cpu().numpy(), st8)
            for i in range(len(files)):
                if st8[i]:
                    assert bool((ints(out[i]) == ints(guard[i])).all()), (dtype, i)
                else:
                    assert bool((ints(out[i].permute(1, 2, 0)) == ints(expect(u8[i], s, b, dtype))).all()), (dtype, i)
    finally:
        gpu.set_decode_verify(False)


# ---- launches and rejections ---------------------------------------------------------------------------------------------
def launches(gpu, fn):
    import torch
    torch.cuda.synchronize()
    before = gpu.launch_count()
    fn()
    torch.cuda.synchronize()
    return gpu.launch_count() - before


def test_typed_calls_launch_like_their_uint8_twins(gpu):
    import torch
    w, h, c = 40, 6, 4
    files = corpus(gpu, w, h, c)[:3]
    t, _, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, device="cuda")
    data, offsets, psizes = packed_device(files)
    for verify in (False, True):
        gpu.set_decode_verify(verify)
        try:
            for d in (3, 4):
                calls = (lambda **k: gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d, **k),
                         lambda **k: gpu.decode_packed_device(data, offsets, psizes, w, h, c, d, **k),
                         lambda dtype=torch.uint8: gpu.decode_packed_ragged_device(
                             data, offsets, psizes, d, max_file_size=1 << 16, max_w=w, max_h=h,
                             out=torch.empty((1 << 14,), dtype=dtype, device="cuda"), dtype=dtype))
                for call in calls:
                    base = launches(gpu, lambda: call())
                    for dtype in DTYPES:
                        assert launches(gpu, lambda: call(dtype=tdt(dtype))) == base, (verify, d, dtype)
        finally:
            gpu.set_decode_verify(False)


def test_typed_calls_reject_bad_arguments(gpu):
    import torch
    from fpng_b200._lib import PixelFormat, lib
    L = lib()
    w, h, c, n, d = 40, 6, 3, 2, 3
    files = corpus(gpu, w, h, c)[:n]
    t, stride, fsz, ofs, lens, *_ = gpu.pack_files_for_device(files, device="cuda")
    fsz, ofs, lens = (np.ascontiguousarray(a, dtype=np.uint32) for a in (fsz, ofs, lens))
    data, offsets, psz = packed_device(files)
    pix = filled((n * h * w * 4 * 2 + 64,), "float32")
    guard = pix.clone()
    status = torch.full((n,), 9, dtype=torch.int32, device="cuda")
    oo = torch.full((n + 1,), 9, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    P = pix.data_ptr()

    def fmt(dtype=1, scale=1.0, bias=0.0):
        f = PixelFormat()
        f.dtype = dtype
        f.scale[:] = [scale] * 4
        f.bias[:] = [bias] * 4
        return C.byref(f)

    def batch(ptr, st, f):
        return L.fpngb_decode_batch_device_typed(t.data_ptr(), stride, fsz.ctypes.data_as(C.c_void_p), ofs.ctypes.data_as(C.c_void_p),
                                                 lens.ctypes.data_as(C.c_void_p), n, w, h, c, d, ptr, *st, f, status.data_ptr(), s)

    def packed(ptr, st, f):
        return L.fpngb_decode_packed_device_typed(data.data_ptr(), offsets.data_ptr(), psz.data_ptr(), n, 1 << 16, w, h, c, d, ptr, *st, f,
                                                  status.data_ptr(), s)

    def ragged(ptr, f, cap=pix.numel() * 4):
        return L.fpngb_decode_packed_ragged_device_typed(data.data_ptr(), data.numel(), offsets.data_ptr(), psz.data_ptr(), n, 1 << 16, w, h,
                                                         d, ptr, cap, oo.data_ptr(), None, f, status.data_ptr(), s)

    tight = lambda es: (h * w * d * es, w * d * es, d * es, es)
    before = gpu.launch_count()
    for call in (batch, packed):
        assert call(P + 2, tight(4), fmt()) == ERR_ALIGNMENT                      # d_out not a multiple of sizeof(float)
        assert call(P + 1, tight(2), fmt(2)) == ERR_ALIGNMENT
        assert call(P, (h * w * d * 4, w * d * 4 + 2, d * 4, 4), fmt()) == ERR_ALIGNMENT   # row pitch
        assert call(P, (h * w * d * 2 + 1, w * d * 2, d * 2, 2), fmt(3)) == ERR_ALIGNMENT  # image stride
        assert call(P, (h * w * d * 4, (w * d - 1) * 4, d * 4, 4), fmt()) == ERR_INVALID_ARG   # rows overlap (in elements)
        assert call(P, (h * w * d * 4, w * 4, 4, 0), fmt()) == ERR_INVALID_ARG            # planar, chan stride 0
        assert call(P, (h * w * d * 4, w * d * 4, 8, 4), fmt()) == ERR_INVALID_ARG        # pixel stride 2 elements
        for bad in (0, 4, 99):
            assert call(P, tight(4), fmt(bad)) == ERR_INVALID_ARG
        assert call(P, tight(4), None) == ERR_INVALID_ARG
        for v in (float("nan"), float("inf"), -float("inf")):
            assert call(P, tight(4), fmt(scale=v)) == ERR_INVALID_ARG
            assert call(P, tight(2), fmt(2, bias=v)) == ERR_INVALID_ARG
    assert ragged(P + 4, fmt()) == ERR_ALIGNMENT                                  # d_out % 16
    assert ragged(P, None) == ERR_INVALID_ARG
    assert ragged(P, fmt(0)) == ERR_INVALID_ARG
    assert ragged(P, fmt(bias=float("nan"))) == ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert bool((ints(pix) == ints(guard)).all()) and bool((status == 9).all()) and bool((oo == 9).all())
    # scale / bias entries at index >= desired_chans are ignored, even when not finite
    f = PixelFormat(); f.dtype = 1; f.scale[:] = [1.0, 1.0, 1.0, float("nan")]; f.bias[:] = [0.0, 0.0, 0.0, float("inf")]
    assert packed(P, tight(4), C.byref(f)) == 0
    torch.cuda.synchronize()
    assert bool((status == 0).all())


# ---- one file whose typed output passes 4 GiB --------------------------------------------------------------------------------
def test_typed_output_past_4gib(gpu):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < (16 << 30):
        pytest.skip("needs 16 GB of free device memory")
    w, h, c = 16384, 32768, 3                                                # 6 GiB of float32
    y = torch.arange(h, device="cuda", dtype=torch.int32)[:, None, None]
    x = torch.arange(w, device="cuda", dtype=torch.int32)[None, :, None]
    ch = torch.arange(c, device="cuda", dtype=torch.int32)[None, None, :]
    img = ((y // 64 * 5 + x // 32 * 3 + ch * 80) % 256).to(torch.uint8)     # runs along x: compresses
    files, sizes = gpu.encode_batch_device(img[None])
    del img
    offsets = torch.zeros((1,), dtype=torch.int64, device="cuda")
    s, b = np.float32(1.0 / 255.0), np.float32(-0.5)
    out, st = gpu.decode_packed_device(files.view(-1), offsets, sizes, w, h, c, c, max_file_size=int(sizes[0]), dtype=torch.float32,
                                       scale=s, bias=b)
    del files
    assert int(st[0]) == 0
    assert out.numel() * 4 > (4 << 30)

    def want(yy, xx):
        v = ((yy[:, None, None] // 64 * 5 + xx[None, :, None] // 32 * 3 + ch * 80) % 256).to(torch.float32)
        return v * torch.tensor(s, device="cuda") + torch.tensor(b, device="cuda")

    last = torch.arange(h - 3, h, device="cuda", dtype=torch.int32)
    allx = torch.arange(w, device="cuda", dtype=torch.int32)
    assert bool((ints(out[0, h - 3:]) == ints(want(last, allx))).all())
    ys = torch.arange(0, h, 997, device="cuda", dtype=torch.int32)
    xs = torch.arange(5, w, 1009, device="cuda", dtype=torch.int32)
    assert bool((ints(out[0, ys.long()][:, xs.long()]) == ints(want(ys, xs))).all())
    del out
