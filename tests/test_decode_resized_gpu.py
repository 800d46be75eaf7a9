"""GPU tests of fpngb_decode_packed_resized_device: packed files of mixed shapes decoded, cropped by a per-file box and resized
into one fixed-size batch.  Expected values are oracle-decoded pixels fed through the numpy model of the resize rule
(test_decode_resized_cpu.py); the identity size and an exact 2x downscale must be bit-exact, and float32 output must agree with
torch's CUDA F.interpolate.  Statuses, their order, untouched output slices of failed files, rejected calls, launch counts,
profiling, stream ordering and overlapping streams are checked as for the ragged decode."""
import zlib

import numpy as np
import pytest

import imagegen
from test_decode_device_gpu import to_device
from test_decode_ragged_gpu import pack_at
from test_decode_resized_cpu import TOL_PLAIN, resize_model

pytestmark = pytest.mark.gpu

INVALID_ARG, NOT_FPNG, CRC, SHAPE_MISMATCH, OUT_OF_SPACE, ADLER, BAD_CROP = 2, 1, 4, 100, 101, 102, 103
SENTINEL = -77.0
MEAN, STD = (0.485, 0.456, 0.406, 0.5), (0.229, 0.224, 0.225, 0.5)


def corpus(oracle, seed=0):
    """mixed shapes, RGB and RGBA, three imagegen kinds; (files, decoded [h, w, 4] per file for d = 4 / [h, w, 3] for d = 3)"""
    shapes = [(1, 1), (5, 3), (37, 53), (224, 224), (333, 517), (640, 96), (17, 250), (1000, 7), (448, 448), (90, 7)]
    files = []
    for j, (w, h) in enumerate(shapes):
        c = 3 + (j % 2)
        kind = ("g1", "g0", "g2")[j % 3]
        files.append(oracle.encode(imagegen.make(kind, w, h, c, seed + j), w, h, c, j % 3 == 1))
    return files


def decoded(oracle, f, d):
    st, px, w, h, _ = oracle.decode(f, d)
    assert st == 0
    return px.reshape(h, w, d)


def random_boxes(rs, dims):
    out = []
    for (w, h) in dims:
        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
        out.append((int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1)), bh, bw))
    return np.array(out, np.int32)


def call(gpu, files, d, size, boxes=None, aa=True, dtype=None, nchw=False, scale=None, bias=None, fill=SENTINEL, **kw):
    import torch
    rs = np.random.RandomState(len(files))
    buf, offs = pack_at(files, rs, True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    n, (H, W) = len(files), size
    dt = dtype or torch.uint8
    if nchw:
        out = torch.full((n, d, H, W), fill, dtype=torch.float32, device="cuda").to(dt).permute(0, 2, 3, 1)
    else:
        out = torch.full((n, H, W, d), fill, dtype=torch.float32, device="cuda").to(dt)
    b = None if boxes is None else torch.from_numpy(np.asarray(boxes, np.int32)).cuda()
    out, info, st = gpu.decode_packed_resized_device(data, offsets, sizes, size, d, boxes=b, antialias=aa, out=out, scale=scale,
                                                     bias=bias, **kw)
    torch.cuda.synchronize()
    return out.float().cpu().numpy(), info.cpu().numpy(), st.cpu().numpy()


def expected(oracle, files, d, size, boxes, aa):
    return [resize_model(decoded(oracle, f, d), size[0], size[1], aa, None if boxes is None else boxes[i]) for i, f in enumerate(files)]


def ulp(dtype, v):
    """the spacing of float16 / bfloat16 values at |v|"""
    import torch
    mant, tiny = {torch.float16: (10, 2.0 ** -14), torch.bfloat16: (7, 2.0 ** -126)}[dtype]
    return 2.0 ** (np.floor(np.log2(np.maximum(np.abs(v), tiny))) - mant)


def check_values(got, want, dtype, s, b):
    """got [H, W, C] of dtype (as float), want the model's [H, W, C] float64 values on the 0-255 scale"""
    import torch
    if dtype in (None, torch.uint8):
        exp = np.clip(np.round(want), 0, 255)                                  # numpy rounds half to even, as cvt.rni
        tie = np.abs(np.abs(want - np.floor(want)) - 0.5) < 2.0 ** -9
        bad = (got != exp) & ~tie
        assert not bad.any(), (np.argwhere(bad)[:4], got[bad][:4], want[bad][:4])
        return
    s = np.asarray(s, np.float64)
    b = np.asarray(b, np.float64)
    w = want * s + b
    tol = 2.0 ** -9 * np.abs(s) + 1e-6 * np.abs(w)
    if dtype != torch.float32:
        tol = tol + ulp(dtype, w)
    d = np.abs(got - w)
    assert (d <= tol).all(), (np.argwhere(d > tol)[:4], got[d > tol][:4], w[d > tol][:4])


# ---- 1. model parity ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["uint8", "float32", "float16", "bfloat16"])
def test_model_parity(gpu, oracle, dtype):
    import torch
    dt = getattr(torch, dtype)
    files = corpus(oracle)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(5)
    for d in (3, 4):
        for size in ((224, 224), (31, 67), (1, 1)):
            for aa in (True, False):
                for boxes in (None, random_boxes(rs, dims)):
                    nchw = bool(rs.randint(0, 2))
                    if dt == torch.uint8:
                        s, b = None, None
                    else:
                        s = (1.0 / (255.0 * np.array(STD[:d]))).astype(np.float32)
                        b = (-np.array(MEAN[:d]) / np.array(STD[:d])).astype(np.float32)
                    got, _, st = call(gpu, files, d, size, boxes, aa, dt, nchw, s, b)
                    assert (st == 0).all(), st
                    want = expected(oracle, files, d, size, boxes, aa)
                    for i in range(len(files)):
                        check_values(got[i], want[i], dt, s, b)


def test_layouts_agree(gpu, oracle):
    """NHWC, NCHW and a strided crop of a larger canvas hold the same values"""
    import torch
    files = corpus(oracle, 3)
    for dt in (torch.uint8, torch.bfloat16):
        a, _, _ = call(gpu, files, 3, (57, 41), dtype=dt)
        b, _, _ = call(gpu, files, 3, (57, 41), dtype=dt, nchw=True)
        assert np.array_equal(a, b)
        canvas = torch.full((len(files), 60, 50, 3), 7, dtype=dt, device="cuda")
        view = canvas[:, 2:59, 5:46, :]
        buf, offs = pack_at(files, np.random.RandomState(0), True)
        data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
        gpu.decode_packed_resized_device(data, offsets, sizes, (57, 41), 3, out=view)
        c = canvas.float().cpu().numpy()
        assert np.array_equal(c[:, 2:59, 5:46, :], a)
        mask = np.ones(c.shape, bool); mask[:, 2:59, 5:46, :] = False
        assert (c[mask] == 7).all()


# ---- 2. bit-exact cases --------------------------------------------------------------------------------------------------------
def test_identity_size_equals_ragged_decode(gpu, oracle):
    import torch
    files = corpus(oracle, 7)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(8)
    buf, offs = pack_at(files, rs, True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    for d in (3, 4):
        for dt in (torch.uint8, torch.float16, torch.float32):
            s, b = (None, None) if dt == torch.uint8 else ([0.5, -2.0, 3.0, 1.0][:d], [1.0, 0.25, -7.0, 0.0][:d])
            out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=dt, scale=s, bias=b)
            views = gpu.ragged_views(out, oo, info, st, d)
            for (bh, bw) in ((1, 1), (16, 16), (7, 5)):
                boxes = np.array([(int(rs.randint(0, h - min(bh, h) + 1)), int(rs.randint(0, w - min(bw, w) + 1)), bh, bw)
                                  for (w, h) in dims], np.int32)
                ok = np.array([bh <= h and bw <= w for (w, h) in dims])
                boxes[~ok] = (0, 0, 1, 1)
                for aa in (True, False):
                    got = torch.empty((len(files), bh, bw, d), dtype=dt, device="cuda")
                    _, _, st2 = gpu.decode_packed_resized_device(data, offsets, sizes, (bh, bw), d, boxes=torch.from_numpy(boxes).cuda(),
                                                                 antialias=aa, out=got, scale=s, bias=b)
                    assert (st2.cpu().numpy() == 0).all()
                    for i in np.flatnonzero(ok):
                        t, l = int(boxes[i, 0]), int(boxes[i, 1])
                        assert torch.equal(got[i], views[i][t:t + bh, l:l + bw]), (d, dt, bh, bw, i)


def test_exact_2x_downscale(gpu, oracle):
    import torch
    files = [oracle.encode(imagegen.make("g2", w, h, c, 1), w, h, c, 0) for (w, h, c) in ((64, 32, 3), (100, 60, 4), (128, 128, 3))]
    for d in (3, 4):
        got, _, st = call(gpu, files, d, (16, 24), boxes=[(0, 0, 32, 48), (10, 2, 32, 48), (50, 70, 32, 48)], aa=False,
                          dtype=torch.float32)
        assert (st == 0).all()
        want = expected(oracle, files, d, (16, 24), [(0, 0, 32, 48), (10, 2, 32, 48), (50, 70, 32, 48)], False)
        for i in range(len(files)):
            assert np.array_equal(got[i], want[i].astype(np.float32)), (d, i)


# ---- 3. torch parity --------------------------------------------------------------------------------------------------------
TOL_CUDA_AA = 5e-3


def test_torch_cuda_parity(gpu, oracle):
    """float32 output with scale 1 and bias 0 against F.interpolate on CUDA over each cropped file.  Antialiased output of width 1
    is included: torch's CUDA kernel agrees with the model there (its CPU kernel does not, test_decode_resized_cpu).  With
    antialiasing torch's CUDA kernel is farther from the model than its CPU kernel: 1.05e-3 on a 224 x 224 output here, up to
    4e-3 on 3840 x 2160 -> 224 x 224 (tools/bench_decode_resized.py), hence TOL_CUDA_AA."""
    import torch
    import torch.nn.functional as F
    files = corpus(oracle, 11)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(12)
    compared = refused = 0
    for size in ((224, 224), (3, 1), (1000, 1), (1, 3)):
        for aa in (True, False):
            boxes = random_boxes(rs, dims)
            got, _, st = call(gpu, files, 3, size, boxes, aa, torch.float32)
            assert (st == 0).all()
            for i, f in enumerate(files):
                t, l, bh, bw = (int(v) for v in boxes[i])
                px = decoded(oracle, f, 3)
                x = torch.from_numpy(px[t:t + bh, l:l + bw]).cuda().permute(2, 0, 1)[None].float()
                try:
                    ref = F.interpolate(x, size=size, mode="bilinear", align_corners=False, antialias=aa)[0].permute(1, 2, 0).cpu().numpy()
                except RuntimeError as e:
                    # torch's CUDA antialias kernel keeps all weights of a CTA in shared memory and refuses large downscales
                    # ("Too much shared memory required"); the resized decode has no such limit: check those against the model
                    assert aa and "shared memory" in str(e), e
                    refused += 1
                    check_values(got[i], resize_model(px, size[0], size[1], aa, boxes[i]), torch.float32, 1.0, 0.0)
                    continue
                compared += 1
                dmax = np.abs(ref - got[i]).max()
                assert dmax <= (TOL_CUDA_AA if aa else TOL_PLAIN), (size, aa, i, dmax)
    assert compared > 3 * refused, (compared, refused)


# ---- 4. statuses ------------------------------------------------------------------------------------------------------------
def test_statuses_and_untouched_slices(gpu, oracle):
    import torch
    enc = lambda k, w, h, c, s: oracle.encode(imagegen.make(k, w, h, c, s), w, h, c, 0)  # noqa: E731
    good = [enc("g1", 64, 16, 4, 1), enc("g0", 33, 7, 3, 2), enc("g1", 120, 30, 3, 3), enc("g2", 48, 48, 4, 4)]
    wide = enc("g1", 200, 8, 3, 5)
    files = [good[0], good[1], good[2], good[3], good[0][:40], wide, good[1], good[2], good[3], good[0], b"", good[1]]
    boxes = np.array([(0, 0, 16, 64), (-1, 0, 3, 3), (0, 0, 30, 0), (40, 40, 9, 8),      # ok, negative top, empty, past the edge
                      (-5, -5, 0, 0), (-5, -5, 0, 0), (0, -1, 2, 2), (0, 100, 30, 21),     # walk and shape win over the box
                      (0, 0, 48, 48), (15, 63, 1, 1), (0, 0, 1, 1), (6, 32, 1, 1)], np.int32)
    walk = gpu.get_info_ex(files[4])[0]
    assert walk not in (0, INVALID_ARG)
    want = [0, BAD_CROP, BAD_CROP, BAD_CROP, walk, SHAPE_MISMATCH, BAD_CROP, BAD_CROP, 0, 0, INVALID_ARG, 0]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=150, max_h=60)
    # BAD_CROP files take no space: pixel_cap of the four good files fits all of them exactly
    cap = sum((w * h * 4 + 15) // 16 * 16 for (w, h) in ((64, 16), (48, 48), (64, 16), (33, 7)))
    got, info, st = call(gpu, files, 4, (9, 13), boxes, True, torch.float32, pixel_cap=cap, **bounds)
    assert st.tolist() == want, st.tolist()
    assert info[4][0] == walk and tuple(info[10]) == (INVALID_ARG, 0, 0, 0, 0, 0)
    for i in range(len(files)):
        if want[i]:
            assert (got[i] == SENTINEL).all(), i
        else:
            exp = resize_model(decoded(oracle, files[i], 4), 9, 13, True, boxes[i])
            check_values(got[i], exp, torch.float32, 1.0, 0.0)
    # one byte less: the last good file gets OUT_OF_SPACE and its slice stays untouched
    got, _, st = call(gpu, files, 4, (9, 13), boxes, True, torch.float32, pixel_cap=cap - 1, **bounds)
    assert st.tolist() == want[:11] + [OUT_OF_SPACE]
    assert (got[11] == SENTINEL).all()


def test_out_of_space_across_placement_rounds(gpu, oracle):
    """n = 1025: the 1024-file placement round boundary; files past pixel_cap keep their sentinel slices"""
    import torch
    f = [oracle.encode(imagegen.make("g1", 9 + k, 5, 3, k), 9 + k, 5, 3, 0) for k in range(5)]
    files = [f[i % 5] for i in range(1025)]
    take = [((9 + (i % 5)) * 5 * 3 + 15) // 16 * 16 for i in range(1025)]
    cut = 1020
    cap = sum(take[:cut])
    bounds = dict(max_file_size=max(len(x) for x in f), max_w=13, max_h=5)
    got, _, st = call(gpu, files, 3, (4, 4), None, True, torch.uint8, fill=99, pixel_cap=cap, **bounds)
    assert (st[:cut] == 0).all() and (st[cut:] == OUT_OF_SPACE).all()
    assert (got[cut:] == 99).all()
    for i in (0, 1000, 1019):
        check_values(got[i], resize_model(decoded(oracle, files[i], 3), 4, 4, True), None, None, None)


def damaged(f, gpu, what):
    """the file with its IDAT CRC field changed (what = "crc"), or with the zlib Adler-32 changed and the IDAT CRC recomputed"""
    _, _, _, _, io, il = gpu.get_info_ex(f)
    b = bytearray(f)
    if what == "crc":
        b[io + 8 + il] ^= 0x10
    else:
        b[io + 8 + il - 1] ^= 0x01
        b[io + 8 + il:io + 12 + il] = zlib.crc32(bytes(b[io + 4:io + 8 + il])).to_bytes(4, "big")
    return bytes(b)


def test_verify_statuses(gpu, oracle):
    import torch
    good = [oracle.encode(imagegen.make("g1", w, h, c, w), w, h, c, 0) for (w, h, c) in ((40, 20, 3), (64, 33, 4), (17, 9, 3))]
    files = [good[0], damaged(good[1], gpu, "crc"), damaged(good[2], gpu, "adler"), good[1], damaged(good[0], gpu, "adler")]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=64, max_h=33, pixel_cap=1 << 20)   # no walk of their own
    before = gpu.launch_count()
    gpu.set_decode_verify(True)
    try:
        got, _, st = call(gpu, files, 3, (8, 8), None, True, torch.float16, **bounds)
    finally:
        gpu.set_decode_verify(False)
    assert gpu.launch_count() - before == 14
    assert st.tolist() == [0, CRC, ADLER, 0, ADLER]
    for i in (1, 2, 4):
        assert (got[i] == SENTINEL).all()
    # verify off: the damaged Adler files decode, the CRC damage is not seen
    before = gpu.launch_count()
    _, _, st = call(gpu, files, 3, (8, 8), None, True, torch.float16, **bounds)
    assert gpu.launch_count() - before == 12 and st.tolist() == [0, 0, 0, 0, 0]


# ---- 5. rejected calls, launches, profiling ----------------------------------------------------------------------------------
def test_rejected_calls(gpu, oracle):
    import torch
    import ctypes as C
    from fpng_b200._lib import PixelFormat, lib
    files = corpus(oracle)[:3]
    buf, offs = pack_at(files, np.random.RandomState(0), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    out = torch.full((3, 8, 8, 4), -5.0, dtype=torch.float32, device="cuda")
    st = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    info = torch.full((3, 6), -7, dtype=torch.int32, device="cuda")
    fmt = PixelFormat(); fmt.dtype = 1; fmt.scale[:] = [1.0] * 4
    bad_fmt = PixelFormat(); bad_fmt.dtype = 9
    nan_fmt = PixelFormat(); nan_fmt.dtype = 1; nan_fmt.scale[:] = [float("nan")] * 4
    o = out.data_ptr()

    def args(**kw):
        a = dict(base=data.data_ptr(), bb=data.numel(), n=3, mfs=1 << 20, mw=1 << 12, mh=1 << 12, cap=1 << 24, boxes=None, ow=8, oh=8,
                 d=4, flags=1, fmt=C.byref(fmt), out=o, strides=(8 * 8 * 16, 8 * 16, 16, 4))
        a.update(kw)
        return (a["base"], a["bb"], offsets.data_ptr(), sizes.data_ptr(), a["n"], a["mfs"], a["mw"], a["mh"], a["cap"], a["boxes"],
                a["ow"], a["oh"], a["d"], a["flags"], a["fmt"], a["out"], *a["strides"], info.data_ptr(), st.data_ptr(), None)

    cases = [(dict(n=0), 1), (dict(n=65536), 1), (dict(ow=0), 1), (dict(oh=0), 1), (dict(ow=(1 << 24) + 1), 1), (dict(oh=(1 << 24) + 1), 1),
             (dict(d=2), 1), (dict(d=5), 1), (dict(flags=2), 1), (dict(fmt=C.byref(bad_fmt)), 1), (dict(fmt=C.byref(nan_fmt)), 1),
             (dict(out=None), 1), (dict(base=None), 1), (dict(mfs=0), 1), (dict(mw=0), 1), (dict(mh=(1 << 24) + 1), 1),
             (dict(strides=(8 * 8 * 16, 8 * 16, 8, 4)), 1), (dict(strides=(8 * 16, 8 * 16, 16, 4)), 1),
             (dict(base=data.data_ptr() + 2), 5), (dict(out=o + 2), 5), (dict(strides=(8 * 8 * 16, 8 * 16 + 2, 16, 4)), 5)]
    before = gpu.launch_count()
    for kw, rc in cases:
        assert lib().fpngb_decode_packed_resized_device(*args(**kw)) == rc, kw
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu().numpy() == -5).all() and (st.cpu().numpy() == -7).all() and (info.cpu().numpy() == -7).all()
    # the same arguments are accepted as they are
    assert lib().fpngb_decode_packed_resized_device(*args()) == 0
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == 0).all() and gpu.launch_count() - before == 12


def test_profile_slot_8(gpu, oracle):
    import torch
    import ctypes as C
    from fpng_b200._lib import lib
    files = corpus(oracle)
    L = lib()
    L.fpngb_decode_profile_enable(1)
    try:
        call(gpu, files, 3, (224, 224), dtype=torch.bfloat16)
        ms = (C.c_float * 9)()
        assert L.fpngb_decode_profile_read(ms, 9) == 1
        assert ms[8] > 0 and ms[6] == 0 and ms[7] == 0 and ms[0] > 0 and ms[5] > 0, list(ms)
        six = (C.c_float * 6)()
        assert L.fpngb_decode_profile_read(six, 6) == 1 and list(six) == list(ms)[:6]
    finally:
        L.fpngb_decode_profile_enable(0)


# ---- 6. stream ordering -----------------------------------------------------------------------------------------------------
def test_no_host_synchronisation(gpu, oracle):
    import torch
    files = corpus(oracle)
    buf, offs = pack_at(files, np.random.RandomState(1), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),
                  pixel_cap=sum((w * h * 4 + 15) // 16 * 16 for w, h in dims))
    out = torch.empty((len(files), 3, 64, 64), dtype=torch.bfloat16, device="cuda").permute(0, 2, 3, 1)
    gpu.decode_packed_resized_device(data, offsets, sizes, (64, 64), 3, out=out, **bounds)     # workspace reserved first
    torch.cuda.synchronize()
    want = out.float().cpu().numpy()
    out.fill_(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (64, 64), 3, out=out, **bounds)
        assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert (st.cpu().numpy() == 0).all() and np.array_equal(out.float().cpu().numpy(), want)


def test_two_streams_with_workspace_growth(gpu, oracle):
    import torch
    small = corpus(oracle)[:4]
    big = [oracle.encode(imagegen.make("g1", 1920, 1080, 3, k), 1920, 1080, 3, 0) for k in range(3)] + corpus(oracle, 20)

    def prep(files):
        buf, offs = pack_at(files, np.random.RandomState(2), True)
        return to_device(buf, offs, [len(f) for f in files])

    A, B = prep(small), prep(big)
    dims_b = [gpu.get_info_ex(f)[1:3] for f in big]
    kw_a = dict(max_file_size=max(len(f) for f in small), max_w=640, max_h=448, pixel_cap=1 << 20)
    kw_b = dict(max_file_size=max(len(f) for f in big), max_w=1920, max_h=1080,
                pixel_cap=sum((w * h * 4 + 15) // 16 * 16 for w, h in dims_b))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for st_ in (s1, s2):
        st_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        torch.cuda._sleep(1 << 28)
        oa, _, sa = gpu.decode_packed_resized_device(*A, (96, 80), 4, dtype=torch.float32, scale=0.5, **kw_a)
    with torch.cuda.stream(s2):
        torch.cuda._sleep(1 << 26)
        ob, _, sb = gpu.decode_packed_resized_device(*B, (224, 224), 3, boxes=None, antialias=False, **kw_b)
    torch.cuda.synchronize()
    alone_a = gpu.decode_packed_resized_device(*A, (96, 80), 4, dtype=torch.float32, scale=0.5, **kw_a)[0].cpu()
    alone_b = gpu.decode_packed_resized_device(*B, (224, 224), 3, boxes=None, antialias=False, **kw_b)[0].cpu()
    assert (sa.cpu().numpy() == 0).all() and (sb.cpu().numpy() == 0).all()
    assert torch.equal(oa.cpu(), alone_a) and torch.equal(ob.cpu(), alone_b)
