"""GPU tests of the native-output any-PNG ragged decode (FPNGB_PNG_NATIVE, native=True): files decoded at their own channel count
and bit depth, as uint8, uint16 or float, to 0 (each file's own), 1, 2, 3 or 4 channels.  Expected values come from the numpy model of
test_decode_native_cpu.py, which is pinned against Pillow, OpenCV and torchvision there."""
import numpy as np
import pytest

import decode_edges as de
import pngenc_workloads as pw
import pngwrite_formats as pf
from test_decode_device_gpu import to_device
from test_decode_native_cpu import fpng_native16, native16, native_out
from test_decode_png_gpu import fpng_file
from test_decode_ragged_gpu import pack_at

pytestmark = pytest.mark.gpu

GUARD = 0xA5
TOO_LARGE, OUT_OF_SPACE = 6, 101
DTYPES = ["uint8", "uint16", "float32"]


def packed(files, seed=0):
    buf, offs = pack_at(files, np.random.RandomState(seed), False)
    return to_device(buf, offs, [len(f) for f in files])


def run(gpu, files, d, dtype="uint8", native=True, all_formats=True, cap=None, seed=0, stream=None, **kw):
    """one ragged call with every bound given (no host sync inside) into a guard-filled output; returns (views, status, info, raw)"""
    import torch
    T = getattr(torch, dtype)
    data, offsets, sizes = packed(files, seed)
    infos = [gpu.get_png_info(f, all_formats=True) for f in files]
    es = torch.empty((), dtype=T).element_size()
    if cap is None:
        cap = max(16, sum((i[1] * i[2] * (d or i[3]) * es + 15) // 16 * 16 for i in infos if i[0] == 0))
    raw = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = raw[:cap].view(T) if es > 1 else raw[:cap]
    _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out, max_file_size=max(len(f) for f in files),
                                                      max_w=max([i[1] for i in infos] + [1]), max_h=max([i[2] for i in infos] + [1]),
                                                      any_png=True, all_formats=all_formats, native=native, stream=stream, **kw)
    torch.cuda.synchronize()
    return gpu.ragged_views(out, oo, info, st, d), st.cpu().numpy(), info.cpu().numpy(), raw


def as_np(v):
    import torch
    return v.cpu().view(torch.int16).numpy().view(np.uint16) if str(v.dtype) == "torch.uint16" else v.cpu().numpy()


# ---- encode -> decode round trip at the image's own shape and dtype -------------------------------------------------------------
def test_round_trip_encode_png_device(gpu):
    import torch
    imgs = [img for _, img in pw.corpus()] + pw.workload("E1", 2) + pw.workload("E2", 2) + pw.workload("E3", 1) + pw.workload("E4", 1)
    imgs += [np.random.default_rng(5).integers(0, 256, (37, 53, c)).astype(np.uint8) for c in (3, 4)]   # fpng files in the same list
    dev = [torch.from_numpy(i.view(np.int16)).view(torch.uint16).cuda() if i.dtype == np.uint16 else torch.from_numpy(i).cuda()
           for i in imgs]
    data, offsets, sizes = gpu.encode_png_device(dev)
    o, z = offsets.cpu().numpy(), sizes.cpu().numpy()
    for dtype in ("uint8", "uint16"):
        sel = [k for k, i in enumerate(imgs) if (i.dtype == np.uint16) == (dtype == "uint16")]
        sub = [data[int(o[k]):int(o[k]) + int(z[k])] for k in sel]
        flat = torch.cat([torch.nn.functional.pad(s, (0, (-s.numel()) % 16)) for s in sub])
        ofs = torch.tensor(np.cumsum([0] + [(s.numel() + 15) // 16 * 16 for s in sub])[:-1], dtype=torch.int64, device="cuda")
        szs = torch.tensor([int(z[k]) for k in sel], dtype=torch.int32, device="cuda")
        px, oo, info, st = gpu.decode_packed_ragged_device(flat, ofs, szs, 0, any_png=True, all_formats=True, native=True,
                                                           dtype=getattr(torch, dtype))
        views = gpu.ragged_views(px, oo, info, st, 0)
        assert not st.any().item()
        for j, k in enumerate(sel):
            assert np.array_equal(as_np(views[j]), imgs[k]), (dtype, k, imgs[k].shape)


# ---- every format, every channel count and dtype ----------------------------------------------------------------------------------
SHAPES = [(1, 1), (2, 3), (5, 4), (9, 7), (17, 1), (13, 17), (33, 5)]


@pytest.mark.parametrize("combo", pf.combos(), ids=lambda c: "t%d_d%d_i%d_%s" % (c[0], c[1], c[2], "trns" if c[3] else "plain"))
def test_every_format(gpu, combo):
    ctype, depth, il, t = combo
    rs = np.random.RandomState(100 * ctype + depth + 7 * il + 3 * t)
    cases = [pf.case(rs, w, h, ctype, depth, il, t, seed=k) for k, (w, h) in enumerate(SHAPES)]
    cases += [pf.case(rs, 19, 11, ctype, depth, il, t, filters=ft, seed=50 + ft) for ft in range(5)]
    for d in (0, 1, 2, 3, 4):
        for dtype in DTYPES:
            views, st, info, raw = run(gpu, [c[0] for c in cases], d, dtype)
            for k, (png, s, plte, trns) in enumerate(cases):
                assert st[k] == 0 and info[k][3] == pf.info_chans(ctype, trns), (k, st[k])
                want = native_out(native16(s, ctype, depth, d, plte, trns), depth, dtype)
                assert np.array_equal(as_np(views[k]), want), (d, dtype, k, s.shape)


def test_float_scale_bias(gpu):
    import torch
    rs = np.random.RandomState(3)
    cases = [(ctype, depth) + pf.case(rs, 11, 6, ctype, depth, 0, False, seed=ctype) for ctype, depth in ((0, 16), (2, 16), (6, 8), (3, 4))]
    for d, sc, bi in ((1, [0.5], [-1.0]), (2, [0.25, 2.0], [1.0, -3.0])):
        for dtype in ("float32", "float16", "bfloat16"):
            views, st, _, _ = run(gpu, [c[2] for c in cases], d, dtype, scale=sc, bias=bi)
            for k, (ctype, depth, png, s, plte, trns) in enumerate(cases):
                m = native16(s, ctype, depth, d, plte, trns)
                x = torch.from_numpy(m.astype(np.float32) / np.float32(257.0) if depth == 16 else (m >> 8).astype(np.float32))
                want = (x * torch.tensor(sc) + torch.tensor(bi)).to(getattr(torch, dtype))
                assert st[k] == 0 and torch.equal(views[k].cpu(), want), (d, dtype, k)


# ---- fpng files -------------------------------------------------------------------------------------------------------------------
def fpng_cases(gpu, oracle):
    import imagegen
    import torch
    out = []
    for k, (w, h, c) in enumerate(((1, 1, 3), (5, 3, 4), (64, 17, 3), (130, 9, 4), (33, 33, 3))):
        png, img = fpng_file(gpu, w, h, c, k)
        out.append((png, img.reshape(h, w, c)))
        img2 = imagegen.make("g1", w, h, c, 10 + k)
        out.append((oracle.encode(img2, w, h, c, 0), img2.reshape(h, w, c)))
    dev_imgs = [torch.from_numpy(np.ascontiguousarray(i)).cuda() for _, i in out[:4]]
    data, offsets, sizes = gpu.encode_png_device(dev_imgs)                  # GPU-written fpng files
    o, s = offsets.cpu().numpy(), sizes.cpu().numpy()
    d = data.cpu().numpy()
    out += [(d[o[k]:o[k] + s[k]].tobytes(), out[k][1]) for k in range(4)]
    return out


def test_fpng_files(gpu, oracle):
    import torch
    cases = fpng_cases(gpu, oracle)
    files = [f for f, _ in cases]
    for d in (3, 4):
        for dtype in ("uint8", "float32"):
            on, st_on, _, _ = run(gpu, files, d, dtype)
            off, st_off, _, _ = run(gpu, files, d, dtype, native=False, **({"scale": 1.0} if dtype != "uint8" else {}))
            assert (st_on == 0).all() and (st_off == 0).all()
            for k in range(len(files)):
                assert torch.equal(on[k].cpu().view(torch.uint8), off[k].cpu().view(torch.uint8)), (d, dtype, k)
    for d in (0, 1, 2):
        views, st, _, _ = run(gpu, files, d)
        assert (st == 0).all()
        for k, (_, img) in enumerate(cases):
            assert np.array_equal(as_np(views[k]), native_out(fpng_native16(img, d), 8, "uint8")), (d, k)
    for d in (0, 1, 2, 3, 4):
        u8, _, _, _ = run(gpu, files, d)
        u16, st, _, _ = run(gpu, files, d, "uint16")
        assert (st == 0).all()
        for k in range(len(files)):
            assert np.array_equal(as_np(u16[k]).astype(np.int64), as_np(u8[k]).astype(np.int64) * 257), (d, k)


def test_flag_on_keeps_3_and_4_channel_bytes(gpu, oracle):
    """a mixed fpng, 8-bit general and ext batch: desired 3 / 4 in uint8 and every float type give the flag-off call's bytes"""
    import torch
    rs = np.random.RandomState(8)
    files = [f for f, _ in fpng_cases(gpu, oracle)[:4]]
    files += [pf.case(rs, 21, 9, ctype, 8, 0, False, seed=ctype)[0] for ctype in (0, 2, 4, 6)]
    files += [pf.case(rs, 13, 12, ctype, depth, il, t, seed=7)[0] for ctype, depth, il, t in ((3, 2, 0, True), (0, 16, 1, True), (6, 16, 0, False))]
    for d in (3, 4):
        for dtype, kw in [("uint8", {})] + [(t, {"scale": [0.5] * d, "bias": [0.25] * d}) for t in ("float32", "float16", "bfloat16")]:
            _, st_on, _, raw_on = run(gpu, files, d, dtype, **kw)
            _, st_off, _, raw_off = run(gpu, files, d, dtype, native=False, **kw)
            assert (st_on == 0).all() and torch.equal(raw_on, raw_off), (d, dtype)


# ---- statuses and placement -------------------------------------------------------------------------------------------------------
def _huge(png):
    """png with its IHDR set to 2^15 x 2^15 (2^30 pixels): its walk passes, its stream is never read"""
    from test_container_cpu import _chunk, _split
    sig, ch = _split(png)
    ihdr = bytearray(ch[0][1]); ihdr[0:4] = (1 << 15).to_bytes(4, "big"); ihdr[4:8] = (1 << 15).to_bytes(4, "big")
    return sig + _chunk(b"IHDR", bytes(ihdr)) + b"".join(c[2] for c in ch[1:])


def test_too_large_uses_file_channels(gpu):
    import torch
    rs = np.random.RandomState(1)
    small = pf.case(rs, 8, 8, 0, 8)[0]
    gray, rgba = _huge(pf.case(rs, 8, 8, 0, 8)[0]), _huge(pf.case(rs, 8, 8, 6, 8)[0])
    files = [small, gray, rgba]
    data, offsets, sizes = packed(files)
    for d, want in ((0, [0, OUT_OF_SPACE, TOO_LARGE]), (1, [0, OUT_OF_SPACE, OUT_OF_SPACE]), (4, [0, TOO_LARGE, TOO_LARGE])):
        out = torch.empty(4096, dtype=torch.uint8, device="cuda")
        _, _, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out, max_file_size=max(map(len, files)),
                                                         max_w=1 << 15, max_h=1 << 15, any_png=True, all_formats=True, native=True)
        assert st.cpu().tolist() == want, (d, st)


def test_out_of_space_two_byte_elements(gpu):
    """uint16 output: a cap one 16-byte unit short of the total leaves the last file OUT_OF_SPACE and its bytes untouched"""
    rs = np.random.RandomState(2)
    cases = [pf.case(rs, w, h, ctype, depth, seed=k) for k, (w, h, ctype, depth) in enumerate(((7, 3, 0, 16), (5, 5, 6, 16), (9, 4, 4, 8)))]
    files = [c[0] for c in cases]
    need = [(w * h * pf.info_chans(c[0], None) * 2 + 15) // 16 * 16 for (w, h, c) in ((7, 3, (0,)), (5, 5, (6,)), (9, 4, (4,)))]
    views, st, _, raw = run(gpu, files, 0, "uint16", cap=sum(need) - 16)
    assert st.tolist() == [0, 0, OUT_OF_SPACE]
    for k in (0, 1):
        png, s, plte, trns = cases[k]
        assert np.array_equal(as_np(views[k]), native_out(native16(s, pf.parse(png)["ctype"], pf.parse(png)["depth"], 0), 16, "uint16"))
    assert (raw[need[0] + need[1]:].cpu().numpy() == GUARD).all()


def test_worst_ratio_tight_cap(gpu):
    """RGBA16 files decoded to 1 channel (8 inflated bytes per output value) at an exactly tight out_cap: every file decodes"""
    rs = np.random.RandomState(4)
    cases = [pf.case(rs, w, h, 6, 16, il, seed=k) for k, (w, h, il) in enumerate(((64, 64, 0), (1, 200, 0), (200, 1, 1), (37, 29, 1), (16, 16, 0)))]
    for dtype in ("uint8", "uint16"):
        views, st, _, raw = run(gpu, [c[0] for c in cases], 1, dtype)
        assert (st == 0).all(), st
        for k, (png, s, plte, trns) in enumerate(cases):
            assert np.array_equal(as_np(views[k]), native_out(native16(s, 6, 16, 1), 16, dtype)), (dtype, k)


def test_failed_files_untouched(gpu):
    rs = np.random.RandomState(6)
    good = pf.case(rs, 9, 9, 2, 16)[0]
    bad = bytearray(pf.case(rs, 9, 9, 2, 16)[0])
    bad[bad.index(b"IDAT") + 4] = 0                                               # zlib CM 0: FAILED_INVALID_IDAT
    views, st, info, raw = run(gpu, [good, bytes(bad), good], 0, "uint16")
    assert st[0] == 0 and st[2] == 0 and st[1] == 8, st
    keep = np.ones(raw.numel(), bool)
    for k in (0, 2):
        at = views[k].data_ptr() - raw.data_ptr()
        keep[at:at + views[k].numel() * 2] = False
    assert (raw.cpu().numpy()[keep] == GUARD).all()


# ---- rejected calls ---------------------------------------------------------------------------------------------------------------
def test_rejected_calls_enqueue_and_write_nothing(gpu):
    import ctypes as C
    import torch
    from fpng_b200._lib import lib
    from fpng_b200.api import PixelFormat
    rs = np.random.RandomState(9)
    files = [pf.case(rs, 8, 8, 0, 16)[0]]
    data, offsets, sizes = packed(files)
    out = torch.full((4096,), GUARD, dtype=torch.uint8, device="cuda")
    oo = torch.full((2,), -7, dtype=torch.int64, device="cuda"); info = torch.full((1, 6), -7, dtype=torch.int32, device="cuda")
    st = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    u16 = PixelFormat(); u16.dtype = 4
    f32 = PixelFormat(); f32.dtype = 1; f32.scale[0] = float("nan")
    base = (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 1, len(files[0]), 8, 8)
    call = lambda d, flags, fmt, o=out.data_ptr(): lib().fpngb_decode_packed_png_device_ex(  # noqa: E731
        *base, d, o, 4096, oo.data_ptr(), info.data_ptr(), flags, fmt, st.data_ptr(), None)
    torch.cuda.synchronize()
    before = gpu.launch_count()
    for d, flags, fmt, rc in ((5, 5, None, 1), (2, 1, None, 1), (0, 1, None, 1), (1, 0, None, 1), (3, 1, C.byref(u16), 1),
                              (3, 0, C.byref(u16), 1), (1, 5, C.byref(f32), 1), (0, 5, C.byref(f32), 1), (3, 2 | 4, None, 1),
                              (3, 0x100 | 4, None, 1)):
        assert call(d, flags, fmt) == rc, (d, flags)
    assert call(1, 5, C.byref(u16), out.data_ptr() + 2) == 5                  # odd uint16 address (not 16-byte aligned)
    assert call(1, 5, None, out.data_ptr() + 8) == 5
    # the typed ragged call keeps rejecting uint16, the device walk the native bit
    assert lib().fpngb_decode_packed_ragged_device_typed(*base, 3, out.data_ptr(), 4096, oo.data_ptr(), info.data_ptr(), C.byref(u16),
                                                         st.data_ptr(), None) == 1
    assert lib().fpngb_get_png_info_batch_device_ex(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), 1, 4, info.data_ptr(), None) == 1
    # the resized call: uint16 and 1 / 2 channels only with FPNGB_RESIZE_NATIVE, which needs FPNGB_RESIZE_ANY_PNG; no desired 0
    rz = lambda d, flags, fmt, o=out.data_ptr(), es=2: lib().fpngb_decode_packed_resized_device(  # noqa: E731
        *base, 4096, None, 4, 4, d, flags, fmt, o, 16 * max(d, 1) * es, 4 * max(d, 1) * es, max(d, 1) * es, es, info.data_ptr(),
        st.data_ptr(), None)
    for d, flags, fmt, rc in ((3, 4, C.byref(u16), 1), (3, 4 | 8, C.byref(u16), 1), (3, 16, C.byref(u16), 1), (1, 16, None, 1),
                              (2, 4, None, 1), (1, 4 | 8, None, 1), (0, 4 | 16, C.byref(u16), 1), (5, 4 | 16, None, 1),
                              (3, 2 | 4 | 16, None, 1), (3, 4 | 16, C.byref(f32), 1)):
        assert rz(d, flags, fmt, es=2 if fmt is not None else 1) == rc, (d, flags)
    assert rz(1, 4 | 16, C.byref(u16), out.data_ptr() + 1) == 5                # odd uint16 address
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu().numpy() == GUARD).all() and (oo.cpu().numpy() == -7).all()
    assert (info.cpu().numpy() == -7).all() and (st.cpu().numpy() == -7).all()


# ---- launches and streams ---------------------------------------------------------------------------------------------------------
def test_launch_counts_match_flag_off(gpu, oracle):
    rs = np.random.RandomState(12)
    files = [f for f, _ in fpng_cases(gpu, oracle)[:3]] + [pf.case(rs, 9, 9, ctype, depth, seed=1)[0] for ctype, depth in ((0, 8), (2, 16))]
    for all_formats in (False, True):
        for d, dtype in ((3, "uint8"), (4, "float32")):
            counts = []
            for native, dd, dt in ((False, d, dtype), (True, d, dtype), (True, 0, "uint16"), (True, 1, "uint8")):
                kw = {"scale": 1.0} if dt == "float32" else {}
                files_ = files if all_formats else files[:4]                    # the 16-bit file needs all_formats
                before = gpu.launch_count()
                run(gpu, files_, dd, dt, native=native, all_formats=all_formats, **kw)
                counts.append(gpu.launch_count() - before)
            assert len(set(counts)) == 1, (all_formats, d, counts)


def test_two_streams_without_host_sync(gpu):
    import torch
    rs = np.random.RandomState(13)
    cases = [pf.case(rs, 40 + k, 30, ctype, depth, k % 2, seed=k) for k, (ctype, depth) in enumerate(((0, 16), (6, 16), (3, 4), (2, 8)) * 4)]
    files = [c[0] for c in cases]
    data, offsets, sizes = packed(files)
    infos = [gpu.get_png_info(f, all_formats=True) for f in files]
    cap = sum((i[1] * i[2] * i[3] * 2 + 15) // 16 * 16 for i in infos)
    bounds = dict(max_file_size=max(map(len, files)), max_w=max(i[1] for i in infos), max_h=max(i[2] for i in infos))
    outs = [torch.empty(cap // 2, dtype=torch.uint16, device="cuda") for _ in range(2)]
    gpu.decode_packed_ragged_device(data, offsets, sizes, 0, out=outs[0], any_png=True, all_formats=True, native=True, **bounds)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    res = []
    for s, o in zip(streams, outs):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            torch.cuda._sleep(1 << 28)
            res.append(gpu.decode_packed_ragged_device(data, offsets, sizes, 0, out=o, any_png=True, all_formats=True, native=True, **bounds))
            assert not s.query(), "the call waited for the stream"
    for s in streams:
        s.synchronize()
    for (o, oo, info, st) in res:
        assert not st.any().item()
        for k, v in enumerate(gpu.ragged_views(o, oo, info, st, 0)):
            png, smp, plte, trns = cases[k]
            f = pf.parse(png)
            assert np.array_equal(as_np(v), native_out(native16(smp, f["ctype"], f["depth"], 0, plte, trns), f["depth"], "uint16")), k


# ---- resized decode with FPNGB_RESIZE_NATIVE --------------------------------------------------------------------------------------
def resized(gpu, files, d, size, dtype="uint16", nchw=False, aa=True, **kw):
    """one native resized call into a guard-filled [n, H, W, d] output (NHWC, or an NCHW permute); returns (float64 array, status)"""
    import torch
    data, offsets, sizes = packed(files, 1)
    n, (H, W) = len(files), size
    T = getattr(torch, dtype)
    shape = (n, d, H, W) if nchw else (n, H, W, d)
    if dtype == "uint16":
        out = torch.full(shape, 0x5A5A, dtype=torch.int16, device="cuda").view(torch.uint16)
    else:
        out = torch.full(shape, -77, dtype=torch.float32, device="cuda").to(T)
    if nchw:
        out = out.permute(0, 2, 3, 1)
    _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, size, d, antialias=aa, out=out, any_png=True, all_formats=True,
                                                native=True, **kw)
    torch.cuda.synchronize()
    v = as_np(out.contiguous()) if dtype == "uint16" else out.float().cpu().numpy()
    return v.astype(np.float64), st.cpu().numpy()


def test_resized_identity_keeps_16_bit_samples(gpu):
    """a 16-bit ramp whose values are not multiples of 257, resized to its own size: every sample comes back exactly"""
    s = ((np.arange(48 * 80, dtype=np.int64) * 37 + 1) % 65536).astype(np.uint32).reshape(48, 80, 1)
    rgb = np.stack([s[..., 0], 65535 - s[..., 0], (s[..., 0] * 5) % 65536], -1).astype(np.uint32)
    files = [pf.make_png(s, 0, 16), pf.make_png(rgb, 2, 16, 1)]
    for aa in (True, False):
        got, st = resized(gpu, files[:1], 1, (48, 80), aa=aa)
        assert (st == 0).all() and np.array_equal(got[0, ..., 0], s[..., 0].astype(np.float64))
        got, st = resized(gpu, files[1:], 3, (48, 80), aa=aa)
        assert (st == 0).all() and np.array_equal(got[0], rgb.astype(np.float64))


RS_CASES = [((0, 16), 53, 37), ((2, 16), 40, 64), ((6, 16), 31, 29), ((4, 16), 20, 70), ((6, 8), 45, 33), ((3, 4), 17, 50), ((0, 8), 64, 64)]


@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", ["uint16", "uint8", "float32"])
def test_resized_matches_float64_model(gpu, d, dtype):
    from test_decode_resized_cpu import resize_model
    from test_decode_resized_gpu import check_values
    import torch
    rs = np.random.RandomState(20 + d)
    cases = [pf.case(rs, w, h, ctype, depth, seed=k) + (ctype, depth) for k, ((ctype, depth), w, h) in enumerate(RS_CASES)]
    sc, bi = ([0.5, 2.0, 1.0, 0.25][:d], [1.0, -3.0, 0.0, 0.5][:d]) if dtype == "float32" else (None, None)
    for size, aa in (((24, 30), True), ((24, 30), False), ((71, 90), True)):
        got, st = resized(gpu, [c[0] for c in cases], d, size, dtype, aa=aa, scale=sc, bias=bi)
        assert (st == 0).all(), st
        for k, (png, s, plte, trns, ctype, depth) in enumerate(cases):
            m16 = native16(s, ctype, depth, d, plte, trns)
            r = resize_model(m16, size[0], size[1], aa)
            if dtype == "uint16":                   # a rounding of some value within the fp32 bound E of r (decode_edges.bound)
                nx, ny = de.taps(m16.shape[0], m16.shape[1], size[0], size[1], aa, np.arange(size[0]))
                E = de.bound(nx[None, :, None], ny[:, None, None], int(m16.max()))
                lo, hi = np.clip(np.round(r - E), 0, 65535), np.clip(np.round(r + E), 0, 65535)
                assert ((got[k] >= lo) & (got[k] <= hi)).all(), (k, size, aa)
            else:
                check_values(got[k], r / 257.0, None if dtype == "uint8" else torch.float32, sc, bi)


def test_resized_layouts_agree(gpu):
    rs = np.random.RandomState(31)
    files = [pf.case(rs, w, h, ctype, depth, seed=k)[0] for k, ((ctype, depth), w, h) in enumerate(RS_CASES)]
    for d in (1, 2, 3, 4):
        for dtype in ("uint16", "float32"):
            a, sa = resized(gpu, files, d, (33, 21), dtype)
            b, sb = resized(gpu, files, d, (33, 21), dtype, nchw=True)
            assert (sa == 0).all() and (sb == 0).all() and np.array_equal(a, b), (d, dtype)


def test_resized_pixel_cap_counts_16_bit_bytes(gpu):
    """pixel_cap is the bytes of the uint16 intermediate: the exact total decodes every file, 16 bytes less leaves the last one out"""
    rs = np.random.RandomState(32)
    cases = [pf.case(rs, w, h, 6, 8, seed=k) for k, (w, h) in enumerate(((9, 7), (13, 5), (4, 4)))]
    files = [c[0] for c in cases]
    total = sum((w * h * 2 * 2 + 15) // 16 * 16 for (w, h) in ((9, 7), (13, 5), (4, 4)))
    bounds = dict(max_file_size=max(map(len, files)), max_w=13, max_h=7)
    _, st = resized(gpu, files, 2, (8, 8), pixel_cap=total, **bounds)
    assert (st == 0).all()
    got, st = resized(gpu, files, 2, (8, 8), pixel_cap=total - 16, **bounds)
    assert st.tolist() == [0, 0, OUT_OF_SPACE]
    assert (got[2] == 0x5A5A).all()


def test_resized_launch_count_matches_flag_off(gpu):
    import torch
    rs = np.random.RandomState(33)
    files = [pf.case(rs, 20, 10, ctype, depth, seed=1)[0] for ctype, depth in ((2, 8), (0, 16), (3, 4))]
    data, offsets, sizes = packed(files)
    counts = []
    for native, dtype in ((False, torch.uint8), (True, torch.uint8), (True, torch.uint16), (False, torch.float32), (True, torch.float32)):
        torch.cuda.synchronize()
        before = gpu.launch_count()
        gpu.decode_packed_resized_device(data, offsets, sizes, (16, 16), 3, dtype=dtype, any_png=True, all_formats=True, native=native,
                                         max_file_size=max(map(len, files)), max_w=20, max_h=10, pixel_cap=1 << 16)
        counts.append(gpu.launch_count() - before)
    torch.cuda.synchronize()
    assert len(set(counts)) == 1, counts
