"""GPU tests of the bicubic resize (FPNGB_RESIZE_BICUBIC, interpolation="bicubic") in the resized and views decodes.  Expected
values are oracle-decoded pixels fed through the numpy model of test_decode_bicubic_cpu.py under check_values' tolerance rules
(ties exempt for uint8); the identity size, a box against the same pixels packed as a file of its own, and every view against the
resized call plus flip and paste must be bit-exact.  Also: torch's CUDA F.interpolate and torchvision's uint8 eval transform,
overshoot, native 16-bit and gray files, statuses, rejected flag combinations, launches and profiling, a tile grid past 65535
and a whole 4K image resized to one pixel."""
import ctypes as C

import numpy as np
import pytest

import imagegen
import pngwrite_formats as pf
from test_decode_bicubic_cpu import bicubic_model
from test_decode_native_cpu import native16
from test_decode_native_gpu import RS_CASES, as_np, resized
from test_decode_resized_cpu import TOL_PLAIN
from test_decode_resized_gpu import (BAD_CROP, INVALID_ARG, OUT_OF_SPACE, SENTINEL, STD, MEAN, TOL_CUDA_AA, call, check_values,
                                     corpus, decoded, random_boxes)
from test_decode_views_gpu import expected_views, packed, random_views, run_views, same, table

pytestmark = pytest.mark.gpu

BICUBIC = 256
SHAPE_MISMATCH = 100


def files_of(oracle, imgs):
    return [oracle.encode(np.ascontiguousarray(x), x.shape[1], x.shape[0], x.shape[2], 0) for x in imgs]


# ---- 1. model parity ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["uint8", "float32", "float16", "bfloat16"])
def test_model_parity(gpu, oracle, dtype):
    """3 and 4 channels, NHWC and NCHW, whole images and random boxes, both antialias settings; the corpus (1x1 to 640x96) and the
    sizes make both up- and downscales"""
    import torch
    T = getattr(torch, dtype)
    files = corpus(oracle, 60)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(61)
    for d in (3, 4):
        for size in ((224, 224), (31, 67), (480, 9), (1, 1)):
            for aa in (True, False):
                boxes = random_boxes(rs, dims) if rs.randint(0, 3) else None
                nchw = bool(rs.randint(0, 2))
                s, b = (None, None) if T == torch.uint8 else ((1.0 / (255.0 * np.array(STD[:d]))).astype(np.float32),
                                                              (-np.array(MEAN[:d]) / np.array(STD[:d])).astype(np.float32))
                got, _, st = call(gpu, files, d, size, boxes, aa, T, nchw, s, b, interpolation="bicubic")
                assert (st == 0).all(), st
                for i, f in enumerate(files):
                    want = bicubic_model(decoded(oracle, f, d), size[0], size[1], aa, None if boxes is None else boxes[i])
                    check_values(got[i], want, T, s, b)


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_native_16_bit_and_gray(gpu, d):
    """native calls on 16-bit, gray, palette and sub-byte files: uint16 output is a rounding of the model's value within 1 (fp32
    sums of 16-bit samples), uint8 and float32 follow check_values on r / 257"""
    import torch
    rs = np.random.RandomState(70 + d)
    cases = [pf.case(rs, w, h, ctype, depth, seed=k) + (ctype, depth) for k, ((ctype, depth), w, h) in enumerate(RS_CASES)]
    files = [c[0] for c in cases]
    for size, aa in (((24, 30), True), ((24, 30), False), ((71, 90), True), ((71, 90), False)):
        for dtype in ("uint16", "uint8", "float32"):
            sc, bi = ([0.5, 2.0, 1.0, 0.25][:d], [1.0, -3.0, 0.0, 0.5][:d]) if dtype == "float32" else (None, None)
            got, st = resized(gpu, files, d, size, dtype, aa=aa, interpolation="bicubic", scale=sc, bias=bi)
            assert (st == 0).all(), st
            for k, (png, s, plte, trns, ctype, depth) in enumerate(cases):
                r = bicubic_model(native16(s, ctype, depth, d, plte, trns), size[0], size[1], aa)
                if dtype == "uint16":
                    lo, hi = np.clip(np.round(r - 1), 0, 65535), np.clip(np.round(r + 1), 0, 65535)
                    assert ((got[k] >= lo) & (got[k] <= hi)).all(), (k, size, aa)
                else:
                    check_values(got[k], r / 257.0, None if dtype == "uint8" else torch.float32, sc, bi)


# ---- 2. bit-exact cases --------------------------------------------------------------------------------------------------------
def test_identity_size_equals_ragged_decode(gpu, oracle):
    """at identity size both filters weigh the source pixel 1 and its neighbours 0: the ragged decode cropped to the box"""
    import torch
    files = corpus(oracle, 62)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(63)
    data, offsets, sizes = packed(files, 1)
    for d in (3, 4):
        for dt in (torch.uint8, torch.float16, torch.float32):
            s, b = (None, None) if dt == torch.uint8 else ([0.5, -2.0, 3.0, 1.0][:d], [1.0, 0.25, -7.0, 0.0][:d])
            out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=dt, scale=s, bias=b)
            views = gpu.ragged_views(out, oo, info, st, d)
            for (bh, bw) in ((1, 1), (16, 16), (7, 5), (33, 40)):
                boxes = np.array([(int(rs.randint(0, h - min(bh, h) + 1)), int(rs.randint(0, w - min(bw, w) + 1)), bh, bw)
                                  for (w, h) in dims], np.int32)
                ok = np.array([bh <= h and bw <= w for (w, h) in dims])
                boxes[~ok] = (0, 0, 1, 1)
                for aa in (True, False):
                    got = torch.empty((len(files), bh, bw, d), dtype=dt, device="cuda")
                    _, _, st2 = gpu.decode_packed_resized_device(data, offsets, sizes, (bh, bw), d, boxes=torch.from_numpy(boxes).cuda(),
                                                                 antialias=aa, out=got, scale=s, bias=b, interpolation="bicubic")
                    assert (st2.cpu().numpy() == 0).all()
                    for i in np.flatnonzero(ok):
                        t, l = int(boxes[i, 0]), int(boxes[i, 1])
                        assert torch.equal(got[i], views[i][t:t + bh, l:l + bw]), (d, dt, bh, bw, aa, i)
    # native uint16: 16-bit samples come back as they are
    smp = ((np.arange(48 * 80, dtype=np.int64) * 37 + 1) % 65536).astype(np.uint32).reshape(48, 80, 1)
    for aa in (True, False):
        got, st = resized(gpu, [pf.make_png(smp, 0, 16)], 1, (48, 80), aa=aa, interpolation="bicubic")
        assert (st == 0).all() and np.array_equal(got[0, ..., 0], smp[..., 0].astype(np.float64))


def test_box_reads_only_the_crop(gpu, oracle):
    """the plain filter's taps past the box read the box's edge pixels, never the file's pixels around it: a box whose surroundings
    are far from its edge pixels equals, bit for bit, the same pixels packed as a file of the box's size"""
    import torch
    rs = np.random.RandomState(64)
    imgs, crops, boxes = [], [], []
    for (h, w, c, bh, bw) in ((60, 70, 3, 20, 30), (40, 33, 4, 13, 9), (9, 9, 3, 3, 3), (100, 50, 4, 1, 48)):
        px = np.zeros((h, w, c), np.uint8)
        if c == 4:
            px[..., 3] = 0
        top, left = int(rs.randint(1, h - bh)), int(rs.randint(1, w - bw))
        inner = rs.randint(200, 256, (bh, bw, c)).astype(np.uint8)
        px[top:top + bh, left:left + bw] = inner
        imgs.append(px)
        crops.append(inner)
        boxes.append((top, left, bh, bw))
    whole, cropped = files_of(oracle, imgs), files_of(oracle, crops)
    for d in (3, 4):
        for T in (torch.uint8, torch.float32, torch.bfloat16):
            for aa in (True, False):
                for size in ((17, 45), (5, 3), (64, 64)):
                    a, _, sa = call(gpu, whole, d, size, boxes, aa, T, interpolation="bicubic")
                    b, _, sb = call(gpu, cropped, d, size, None, aa, T, interpolation="bicubic")
                    assert (sa == 0).all() and (sb == 0).all()
                    assert np.array_equal(a, b), (d, T, aa, size)


# ---- 3. torch and torchvision parity ---------------------------------------------------------------------------------------------
def test_torch_cuda_parity(gpu, oracle):
    """float32 output with scale 1 and bias 0 against F.interpolate(mode="bicubic") on CUDA over each cropped file.  The
    tolerances are the bilinear test's: TOL_CUDA_AA with antialiasing (torch's CUDA antialias kernel computes its weights and sums
    in another order), TOL_PLAIN without (torch's tap fraction is rounded differently at large source indices).  torch's CUDA
    antialias kernel refuses large downscales ("Too much shared memory"): those cases are checked against the model."""
    import torch
    import torch.nn.functional as F
    files = corpus(oracle, 65)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(66)
    compared = refused = 0
    worst = {True: 0.0, False: 0.0}
    for size in ((224, 224), (3, 1), (1000, 1), (1, 3), (40, 50)):
        for aa in (True, False):
            boxes = random_boxes(rs, dims)
            got, _, st = call(gpu, files, 3, size, boxes, aa, torch.float32, interpolation="bicubic")
            assert (st == 0).all()
            for i, f in enumerate(files):
                t, l, bh, bw = (int(v) for v in boxes[i])
                px = decoded(oracle, f, 3)
                x = torch.from_numpy(px[t:t + bh, l:l + bw]).cuda().permute(2, 0, 1)[None].float()
                try:
                    ref = F.interpolate(x, size=size, mode="bicubic", align_corners=False, antialias=aa)[0].permute(1, 2, 0).cpu().numpy()
                except RuntimeError as e:
                    assert aa and "shared memory" in str(e), e
                    refused += 1
                    check_values(got[i], bicubic_model(px, size[0], size[1], aa, boxes[i]), torch.float32, 1.0, 0.0)
                    continue
                compared += 1
                dmax = float(np.abs(ref - got[i]).max())
                worst[aa] = max(worst[aa], dmax)
                assert dmax <= (TOL_CUDA_AA if aa else TOL_PLAIN), (size, aa, i, dmax)
    assert compared > 3 * refused, (compared, refused)
    print("bicubic vs torch CUDA, max |diff|: antialias", worst[True], "plain", worst[False])


def test_uint8_eval_transform_matches_torchvision(gpu, oracle):
    """CLIP's eval transform in uint8: resize_crop_views(info, 224, 224) with bicubic antialiased views against torchvision v2's
    resize(224, BICUBIC, antialias=True) + center_crop(224) on a CUDA uint8 tensor (float interpolate, clamp, round).  Pixels whose
    float value sits within TOL_CUDA_AA of a rounding tie are exempt."""
    import torch
    import torchvision.transforms.v2.functional as TF
    from torchvision.transforms import InterpolationMode
    files = corpus(oracle, 67)
    data, offsets, sizes = packed(files)
    info = gpu.get_info_batch_device(data, offsets, sizes)
    views = gpu.resize_crop_views(info, 224, 224)
    got, _, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, views, (224, 224), 3, interpolation="bicubic", antialias=True)
    assert (vst.cpu() == 0).all()
    compared = 0
    for i, f in enumerate(files):
        x = torch.from_numpy(decoded(oracle, f, 3)).cuda().permute(2, 0, 1)
        try:
            ref = TF.center_crop(TF.resize(x, 224, InterpolationMode.BICUBIC, antialias=True), [224, 224]).permute(1, 2, 0)
            flt = TF.center_crop(TF.resize(x.float(), 224, InterpolationMode.BICUBIC, antialias=True), [224, 224]).permute(1, 2, 0)
        except RuntimeError as e:
            assert "shared memory" in str(e), e
            continue
        compared += 1
        frac = (flt - flt.floor() - 0.5).abs()
        bad = (ref != got[i]) & ~((frac < TOL_CUDA_AA) & (flt > -0.5) & (flt < 255.5))
        assert not bad.any(), (i, int(bad.sum()))
    assert compared >= len(files) - 1


def test_overshoot_saturates_uint8_and_stays_in_float(gpu, oracle):
    """a step and a checkerboard: the model leaves [0, 255] on both sides; uint8 output holds 0 and 255 there, float32 output
    holds values below 0 and above 255"""
    import torch
    step = np.zeros((16, 24, 3), np.uint8)
    step[:, 12:] = 255
    board = ((np.indices((12, 12)).sum(0) % 2) * 255).astype(np.uint8)[..., None].repeat(3, 2)
    files = files_of(oracle, [step, board])
    for aa in (True, False):
        for size in ((16, 61), (29, 29)):
            u8, _, st = call(gpu, files, 3, size, None, aa, torch.uint8, interpolation="bicubic")
            f32, _, st2 = call(gpu, files, 3, size, None, aa, torch.float32, interpolation="bicubic")
            assert (st == 0).all() and (st2 == 0).all()
            for i, x in enumerate((step, board)):
                want = bicubic_model(x, size[0], size[1], aa)
                lo, hi = want < -0.5, want > 255.5
                assert lo.any() and hi.any(), (i, aa, size)
                assert (u8[i][lo] == 0).all() and (u8[i][hi] == 255).all()
                assert f32[i].min() < 0 and f32[i].max() > 255
                check_values(u8[i], want, torch.uint8, None, None)
                check_values(f32[i], want, torch.float32, 1.0, 0.0)


# ---- 4. views -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["uint8", "float32", "bfloat16"])
def test_views_equal_resized_flip_paste(gpu, oracle, dtype):
    import torch
    T = getattr(torch, dtype)
    files = corpus(oracle, 68)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(69)
    k = 0
    for d in (3, 4):
        for aa in (True, False):
            layout = ("nhwc", "nchw", "strided")[k % 3]
            canvas = ((64, 80), (33, 17), (1, 1), (96, 96))[k % 4]
            k += 1
            rows = random_views(rs, dims, canvas)
            fill = [int(v) for v in rs.randint(0, 256, d)]
            kw = dict(antialias=aa, interpolation="bicubic")
            if T != torch.uint8:
                kw.update(scale=[0.5, -2.0, 1.0 / 255, 3.0][:d], bias=[1.0, 0.25, -0.5, 0.0][:d])
            pk, got, st, vst = run_views(gpu, files, rows, canvas, d, T, layout, fill, **kw)
            assert (st.cpu() == 0).all() and (vst.cpu() == 0).all(), (st, vst)
            want = expected_views(gpu, *pk, rows, canvas, d, T, fill, kw)
            for v in range(len(rows)):
                assert same(got[v], want[v]), (dtype, d, aa, layout, rows[v])


def test_native_views(gpu):
    import torch
    rs = np.random.RandomState(71)
    files = [pf.case(rs, int(rs.randint(2, 80)), int(rs.randint(2, 50)), ct, dp, il, t, seed=k)[0]
             for k, (ct, dp, il, t) in enumerate([(0, 16, 0, False), (2, 16, 1, True), (6, 8, 0, False), (3, 4, 1, True)])]
    dims = [gpu.get_png_info(f, all_formats=True)[1:3] for f in files]
    for d in (1, 4):
        for T, fill, kw in ((torch.uint16, 40000, {}), (torch.float32, 1000, dict(scale=0.5, bias=-1.0))):
            for aa in (True, False):
                rows = random_views(rs, dims, (23, 31))
                kw2 = dict(any_png=True, all_formats=True, native=True, antialias=aa, interpolation="bicubic", **kw)
                pk, got, st, vst = run_views(gpu, files, rows, (23, 31), d, T, ("nchw", "nhwc")[d % 2], fill, **kw2)
                assert (vst.cpu() == 0).all(), vst
                want = expected_views(gpu, *pk, rows, (23, 31), d, T, fill, kw2)
                for v in range(len(rows)):
                    assert same(got[v], want[v]), (d, T, aa, rows[v])


# ---- 5. statuses, rejected calls, launches ---------------------------------------------------------------------------------------
def test_statuses_and_untouched_slices(gpu, oracle):
    import torch
    enc = lambda k, w, h, c, s: oracle.encode(imagegen.make(k, w, h, c, s), w, h, c, 0)  # noqa: E731
    good = [enc("g1", 64, 16, 4, 1), enc("g0", 33, 7, 3, 2), enc("g1", 120, 30, 3, 3), enc("g2", 48, 48, 4, 4)]
    wide = enc("g1", 200, 8, 3, 5)
    files = [good[0], good[1], good[2], good[3], good[0][:40], wide, good[1], good[2], good[3], good[0], b"", good[1]]
    boxes = np.array([(0, 0, 16, 64), (-1, 0, 3, 3), (0, 0, 30, 0), (40, 40, 9, 8), (-5, -5, 0, 0), (-5, -5, 0, 0), (0, -1, 2, 2),
                      (0, 100, 30, 21), (0, 0, 48, 48), (15, 63, 1, 1), (0, 0, 1, 1), (6, 32, 1, 1)], np.int32)
    walk = gpu.get_info_ex(files[4])[0]
    want = [0, BAD_CROP, BAD_CROP, BAD_CROP, walk, SHAPE_MISMATCH, BAD_CROP, BAD_CROP, 0, 0, INVALID_ARG, 0]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=150, max_h=60)
    cap = sum((w * h * 4 + 15) // 16 * 16 for (w, h) in ((64, 16), (48, 48), (64, 16), (33, 7)))
    for aa in (True, False):
        got, info, st = call(gpu, files, 4, (9, 13), boxes, aa, torch.float32, pixel_cap=cap, interpolation="bicubic", **bounds)
        assert st.tolist() == want, st.tolist()
        for i in range(len(files)):
            if want[i]:
                assert (got[i] == SENTINEL).all(), i
            else:
                check_values(got[i], bicubic_model(decoded(oracle, files[i], 4), 9, 13, aa, boxes[i]), torch.float32, 1.0, 0.0)
        got, _, st = call(gpu, files, 4, (9, 13), boxes, aa, torch.float32, pixel_cap=cap - 1, interpolation="bicubic", **bounds)
        assert st.tolist() == want[:11] + [OUT_OF_SPACE]
        assert (got[11] == SENTINEL).all()


def test_rejected_flag_combinations(gpu, oracle):
    """bicubic with a nearest mode or the index mode: FPNGB_ERR_INVALID_ARG from both C calls, nothing enqueued or written;
    ValueError from Python.  Bicubic with every other flag is accepted, with the bilinear call's launch count."""
    import torch
    from fpng_b200._lib import PixelFormat, lib
    files = corpus(oracle)[:3]
    data, offsets, sizes = packed(files)
    views = table([(i, 0, 0, 1, 1, 8, 8, 0, 0, 0) for i in range(3)])
    out = torch.full((3, 8, 8, 4), -5.0, dtype=torch.float32, device="cuda")
    st = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    vst = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    info = torch.full((3, 6), -7, dtype=torch.int32, device="cuda")
    fmt = PixelFormat(); fmt.dtype = 1; fmt.scale[:] = [1.0] * 4
    u16 = PixelFormat(); u16.dtype = 4
    full = 4 | 8 | 16

    def resized_args(flags, f=fmt, d=4, strides=(8 * 8 * 16, 8 * 16, 16, 4)):
        return (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 3, 1 << 20, 1 << 12, 1 << 12, 1 << 24, None, 8, 8,
                d, flags, f, out.data_ptr(), *strides, info.data_ptr(), st.data_ptr(), None)

    def views_args(flags, f=fmt, d=4, strides=(8 * 8 * 16, 8 * 16, 16, 4)):
        return (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 3, 1 << 20, 1 << 12, 1 << 12, 1 << 24,
                views.data_ptr(), 3, 8, 8, d, flags, f, None, out.data_ptr(), *strides, info.data_ptr(), st.data_ptr(), vst.data_ptr(), None)

    u16_strides = (8 * 8 * 2, 8 * 2, 2, 2)
    bad = [(BICUBIC | 32, C.byref(fmt), 4, None), (BICUBIC | 64, C.byref(fmt), 4, None), (BICUBIC | 32 | 1, C.byref(fmt), 4, None),
           (BICUBIC | full | 128 | 32, C.byref(u16), 1, u16_strides), (BICUBIC | full | 128, C.byref(u16), 1, u16_strides),
           (BICUBIC | 2, C.byref(fmt), 4, None), (BICUBIC | 512, C.byref(fmt), 4, None)]
    before = gpu.launch_count()
    for flags, f, d, strides in bad:
        kw = dict(f=f, d=d) if strides is None else dict(f=f, d=d, strides=strides)
        assert lib().fpngb_decode_packed_resized_device(*resized_args(flags, **kw)) == 1, flags
        assert lib().fpngb_decode_packed_views_device(*views_args(flags, **kw)) == 1, flags
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu() == -5).all() and (st.cpu() == -7).all() and (vst.cpu() == -7).all() and (info.cpu() == -7).all()
    for flags, n in ((BICUBIC, 12), (BICUBIC | 1, 12), (BICUBIC | 1 | 4, 15), (BICUBIC | full, 16)):
        for fn, args in ((lib().fpngb_decode_packed_resized_device, resized_args), (lib().fpngb_decode_packed_views_device, views_args)):
            b = gpu.launch_count()
            assert fn(*args(flags)) == 0, flags
            torch.cuda.synchronize()
            assert gpu.launch_count() - b == n and (st.cpu() == 0).all(), flags
    with pytest.raises(ValueError):
        gpu.decode_packed_resized_device(data, offsets, sizes, (8, 8), 1, interpolation="bicubic", indices=True, any_png=True,
                                         all_formats=True, native=True)
    with pytest.raises(ValueError):
        gpu.decode_packed_views_device(data, offsets, sizes, views, (8, 8), 1, interpolation="bicubic", indices=True, any_png=True,
                                       all_formats=True, native=True)


def test_launches_verify_and_profile_slot_8(gpu, oracle):
    import torch
    from fpng_b200._lib import lib
    files = corpus(oracle)
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=1024, max_h=1024, pixel_cap=1 << 24)
    for verify, n in ((False, 12), (True, 14)):
        gpu.set_decode_verify(verify)
        try:
            for aa in (True, False):
                b = gpu.launch_count()
                _, _, st = call(gpu, files, 3, (32, 32), None, aa, torch.uint8, interpolation="bicubic", **bounds)
                assert gpu.launch_count() - b == n and (st == 0).all()
        finally:
            gpu.set_decode_verify(False)
    L = lib()
    L.fpngb_decode_profile_enable(1)
    try:
        call(gpu, files, 3, (224, 224), dtype=torch.bfloat16, interpolation="bicubic")
        ms = (C.c_float * 9)()
        assert L.fpngb_decode_profile_read(ms, 9) == 1
        assert ms[8] > 0 and ms[6] == 0 and ms[7] == 0 and ms[0] > 0 and ms[5] > 0, list(ms)
    finally:
        L.fpngb_decode_profile_enable(0)


# ---- 6. grid and tap-count edges ---------------------------------------------------------------------------------------------
def test_tile_grid_past_65535(gpu, oracle):
    """a 2 x (2^21 + 100) output has 65 540 tiles of 32 x 32: the tile loop runs past the grid's 65 535 CTAs"""
    import torch
    rs = np.random.RandomState(72)
    x = rs.randint(0, 256, (5, 7, 3)).astype(np.uint8)
    files = files_of(oracle, [x])
    W = (1 << 21) + 100
    for aa in (True, False):
        data, offsets, sizes = packed(files)
        out, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (2, W), 3, antialias=aa, dtype=torch.float32,
                                                      interpolation="bicubic")
        assert (st.cpu() == 0).all()
        want = bicubic_model(x, 2, W, aa)
        got = out[0].cpu().numpy()
        check_values(got, want, torch.float32, 1.0, 0.0)
        del out


def test_whole_4k_to_one_pixel(gpu, oracle):
    """a whole 3840 x 2160 image resized to 1 x 1 with antialias: 7680 x 4320 taps, every source pixel weighted"""
    import torch
    img = imagegen.gradient_noise(3840, 2160, 3, 9)
    files = [oracle.encode(img, 3840, 2160, 3, 0)]
    px = np.asarray(img).reshape(2160, 3840, 3)
    want = bicubic_model(px, 1, 1, True)
    for T in (torch.uint8, torch.float32):
        got, _, st = call(gpu, files, 3, (1, 1), None, True, T, interpolation="bicubic")
        assert (st == 0).all()
        check_values(got[0], want, T, 1.0, 0.0)
