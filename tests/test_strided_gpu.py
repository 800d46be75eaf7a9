"""GPU tests of strided device tensors: encode_batch_device on interleaved rows at any pitch and on planar (CHW / HCW) views,
decode_batch_device / decode_packed_device writing into such views.  Every encode must equal the oracle's bytes and the
encode of the .contiguous() copy; every decode must equal the oracle's pixels and leave every byte outside the view alone."""
import ctypes as C

import numpy as np
import pytest

import imagegen
from test_decode_device_gpu import packed_device
from test_encode_gpu import rows_per_warp  # noqa: F401  (fixture)
from test_trained_tables_cpu import load_tables

pytestmark = pytest.mark.gpu

WIDTHS = [1, 15, 16, 687, 1920, 8192]
FLAGS = (0, 1, 2)                                  # 0, FPNG_ENCODE_SLOWER, FPNG_FORCE_UNCOMPRESSED
GUARD = 0xA5


def files_of(out, sizes):
    sizes = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    out = out.cpu().numpy()
    return [out[i, : sizes[i]].tobytes() for i in range(len(sizes))]


def check_encode(gpu, oracle, view, flags, what=""):
    """encode of the view == encode of its contiguous copy == the oracle, file by file; returns the files"""
    n, h, w, c = view.shape
    got = files_of(*gpu.encode_batch_device(view, flags))
    assert got == files_of(*gpu.encode_batch_device(view.contiguous(), flags)), (what, n, h, w, c, flags)
    host = view.cpu().numpy()
    for i in range(n):
        assert got[i] == oracle.encode(host[i], w, h, c, flags), (what, i, h, w, c, flags)
    return got


def images(kind, n, w, h, c, seed):
    return np.stack([imagegen.make(kind, w, h, c, seed + i) for i in range(n)])


# ---- encode: interleaved rows at any pitch -------------------------------------------------------------------------------
@pytest.mark.parametrize("rows_per_warp", [1, 5], indirect=True)
@pytest.mark.parametrize("c", [3, 4])
def test_encode_interleaved_crops(gpu, oracle, c, rows_per_warp):
    import torch
    for w in WIDTHS:
        h = 3 if w < 8192 else 2
        canvas = torch.from_numpy(images("g1", 2, w + 16, h + 2, c, w)).cuda()
        for x0 in range(16):
            view = canvas[:, 1:1 + h, x0:x0 + w, :]
            for flags in FLAGS:
                check_encode(gpu, oracle, view, flags, ("crop", x0))


# ---- encode: planar ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows_per_warp", [1, 5], indirect=True)
@pytest.mark.parametrize("c", [3, 4])
def test_encode_planar(gpu, oracle, c, rows_per_warp):
    import torch
    for w in WIDTHS:
        h = 5 if w < 8192 else 2
        src = images("g1", 2, w, h, c, 7 * w)
        nchw = torch.from_numpy(np.ascontiguousarray(src.transpose(0, 3, 1, 2))).cuda()
        hcw = torch.from_numpy(np.ascontiguousarray(src.transpose(0, 1, 3, 2))).cuda()
        four = torch.from_numpy(np.ascontiguousarray(images("runs", 2, w, h, 4, w).transpose(0, 3, 1, 2))).cuda()
        for flags in FLAGS:
            check_encode(gpu, oracle, nchw.permute(0, 2, 3, 1), flags, "nchw")
            check_encode(gpu, oracle, hcw.permute(0, 1, 3, 2), flags, "hcw")
            check_encode(gpu, oracle, four[:, 4 - c:].permute(0, 2, 3, 1), flags, "planes of 4")
            for extra, ofs in ((1, 0), (3, 1), (5, 2)):                  # plane strides that are not 4- or 16-byte aligned
                cs = h * w + extra
                flat = torch.full((2 * c * cs + ofs + 16,), 0x5A, dtype=torch.uint8, device="cuda")
                view = flat.as_strided((2, h, w, c), (c * cs, w, 1, cs), ofs)
                view.copy_(torch.from_numpy(src).cuda())
                check_encode(gpu, oracle, view, flags, ("odd planes", extra, ofs))


def test_encode_stored_fallback_both_layouts(gpu, oracle):
    """incompressible images: the stored-block rows are copied from the view in PNG byte order"""
    import torch
    for c in (3, 4):
        for (w, h) in ((687, 9), (1920, 4), (16, 3)):
            src = images("g2", 2, w, h, c, 3)                                 # random bytes
            for flags in (0, 1):
                files = check_encode(gpu, oracle, torch.from_numpy(np.ascontiguousarray(src.transpose(0, 3, 1, 2))).cuda().permute(0, 2, 3, 1),
                                     flags, "stored planar")
                raw = (w * c + 1) * h
                assert all(len(f) >= raw for f in files), "expected the stored-block fallback"
                canvas = torch.zeros((2, h, w + 5, c), dtype=torch.uint8, device="cuda")
                canvas[:, :, 3:3 + w] = torch.from_numpy(src).cuda()
                check_encode(gpu, oracle, canvas[:, :, 3:3 + w], flags, "stored pitched")


def test_encode_tiles_one_call_per_tile_row(gpu, oracle):
    """a 1000 x 700 canvas cut into 256 x 256 tiles: per tile row one call for the full tiles (image_stride = tile_w * chans)
    and one for the edge tile; every file equals the oracle's encode of that crop"""
    import torch
    W, H, T = 1000, 700, 256
    for c in (3, 4):
        host = imagegen.make("g1", W, H, c, 11).reshape(H, W, c)
        canvas = torch.from_numpy(host).cuda()
        for y0 in range(0, H, T):
            th = min(T, H - y0)
            full = W // T
            tiles = canvas.as_strided((full, th, T, c), (T * c, W * c, c, 1), y0 * W * c)
            got = files_of(*gpu.encode_batch_device(tiles, 0))
            for k in range(full):
                assert got[k] == oracle.encode(np.ascontiguousarray(host[y0:y0 + th, k * T:(k + 1) * T]), T, th, c, 0), (c, y0, k)
            edge = canvas[None, y0:y0 + th, full * T:]
            got = files_of(*gpu.encode_batch_device(edge, 0))
            assert got[0] == oracle.encode(np.ascontiguousarray(host[y0:y0 + th, full * T:]), W - full * T, th, c, 0), (c, y0)


def test_encode_broadcast_batch(gpu, oracle):
    import torch
    for c in (3, 4):
        img = torch.from_numpy(imagegen.make("g1", 300, 40, c, 5).reshape(1, 40, 300, c)).cuda()
        for view in (img.expand(6, -1, -1, -1), img.permute(0, 3, 1, 2).contiguous().expand(6, -1, -1, -1).permute(0, 2, 3, 1)):
            got = check_encode(gpu, oracle, view, 0, "expand")
            assert len(set(got)) == 1


# ---- encode: launches and the rare paths ---------------------------------------------------------------------------------
def launches(gpu, fn):
    import torch
    torch.cuda.synchronize()
    before = gpu.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return gpu.launch_count() - before, r


def test_default_path_strided_launches_no_extra_kernel(gpu):
    import torch
    src = torch.from_numpy(images("g1", 3, 200, 20, 3, 1)).cuda()
    nchw = src.permute(0, 3, 1, 2).contiguous()
    crop = torch.zeros((3, 20, 205, 3), dtype=torch.uint8, device="cuda"); crop[:, :, 5:] = src
    for flags in (0, 1):
        base, ref = launches(gpu, lambda: files_of(*gpu.encode_batch_device(src, flags)))
        for view in (nchw.permute(0, 2, 3, 1), crop[:, :, 5:]):
            k, got = launches(gpu, lambda: files_of(*gpu.encode_batch_device(view, flags)))
            assert k == base and got == ref, (flags, k, base)


def test_trained_table_rule_reads_strided_input_in_place(gpu, oracle):
    """RGBA 1-pass under a trained table whose one-pixel-match rule fires reads planar and cropped views in place, as under the
    shipped table: no extra kernel, with byte parity"""
    import torch
    t = load_tables()["4"]
    prefix = bytes.fromhex(t["prefix"])
    sizes = np.array(t["sizes"], np.uint8)
    assert oracle.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
    try:
        gpu.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
        w, h = 61, 24
        pal = [int(v) for v in np.argsort(sizes[:256], kind="stable")[:4]]
        src = np.stack([imagegen.short_runs(w, h, 4, 7 + i, pal) for i in range(4)])
        dev = torch.from_numpy(src).cuda()
        base, ref = launches(gpu, lambda: files_of(*gpu.encode_batch_device(dev, 0)))
        for i in range(4):
            assert ref[i] == oracle.encode(src[i], w, h, 4, 0), i
        planar = dev.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
        canvas = torch.zeros((4, h, w + 3, 4), dtype=torch.uint8, device="cuda"); canvas[:, :, 3:] = dev
        for view in (planar, canvas[:, :, 3:]):
            k, got = launches(gpu, lambda: files_of(*gpu.encode_batch_device(view, 0)))
            assert got == ref and k == base, (k, base)
    finally:
        gpu.set_static_table(4)
        oracle.set_static_table(4)


def test_fused_encoder_gathers_strided_input(gpu, oracle):
    import torch
    from fpng_b200._lib import lib
    L = lib()
    try:
        L.fpngb_debug_use_fused(1)
        for c in (3, 4):
            src = torch.from_numpy(images("g1", 3, 640, 30, c, 2)).cuda()
            planar = src.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
            canvas = torch.zeros((3, 30, 647, c), dtype=torch.uint8, device="cuda"); canvas[:, :, 7:] = src
            for flags in (0, 1):
                check_encode(gpu, oracle, planar, flags, "fused planar")
                check_encode(gpu, oracle, canvas[:, :, 7:], flags, "fused crop")
                # exactly one gather kernel in front of the contiguous call's launches, and the single-pass encoder ran: the
                # per-kernel profile has a single-pass slot and no scan slot
                base, _ = launches(gpu, lambda: gpu.encode_batch_device(src, flags))
                for view in (planar, canvas[:, :, 7:]):
                    ms = (C.c_float * 9)()
                    L.fpngb_profile_read(ms, 9)                                    # drop earlier calls
                    L.fpngb_profile_enable(1)
                    try:
                        k, _ = launches(gpu, lambda: gpu.encode_batch_device(view, flags))
                        assert L.fpngb_profile_read(ms, 9) == 1
                    finally:
                        L.fpngb_profile_enable(0)
                    assert k == base + 1, (c, flags, k, base)
                    assert ms[4] > 0 and ms[2] == 0, (c, flags, list(ms))          # slots: hist, huffman, scan, offsets, fused, ...
    finally:
        L.fpngb_debug_use_fused(-1)


# ---- decode into strided outputs -----------------------------------------------------------------------------------------
def decode_corpus(oracle, w, h, c):
    files = [oracle.encode(imagegen.make(k, w, h, c, 40 + i), w, h, c, flags)
             for i, k in enumerate(("g1", "runs", "g0")) for flags in (0, 1, 2)]
    bad = bytearray(files[0]); bad[58] ^= 0x01                                # zlib header (the walk does not read it): NOT_FPNG
    return files + [bytes(bad)]


def windows(n, h, w, d):
    """(guard-filled buffer, [n, h, w, d] view into it) for a pitched HWC window and for NCHW planes"""
    import torch
    hwc = torch.full((n, h + 2, w + 3, d), GUARD, dtype=torch.uint8, device="cuda")
    yield "hwc", hwc, hwc[:, 1:1 + h, 2:2 + w, :]
    planes = torch.full((n, d + 1, h + 1, w + 2), GUARD, dtype=torch.uint8, device="cuda")
    yield "nchw", planes, planes[:, :d, :h, 1:1 + w].permute(0, 2, 3, 1)
    odd = torch.full((n * (d * (h * w + 3)) + 8,), GUARD, dtype=torch.uint8, device="cuda")
    cs = h * w + 3
    yield "odd planes", odd, odd.as_strided((n, h, w, d), (d * cs, w, 1, cs), 1)


@pytest.mark.parametrize("c", [3, 4])
@pytest.mark.parametrize("d", [3, 4])
def test_decode_into_strided_outputs(gpu, oracle, c, d):
    import torch
    for (w, h) in ((1, 5), (15, 3), (687, 11), (1920, 6)):
        files = decode_corpus(oracle, w, h, c)
        n = len(files)
        expect = []
        for f in files:
            st, px, *_ = oracle.decode(f, d)
            expect.append(px if st == 0 else None)
        assert expect[-1] is None
        t, _, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, device="cuda")
        data, offsets, psizes = packed_device(files)
        # a file of another shape in the packed call: FPNGB_DECODE_SHAPE_MISMATCH, region untouched
        other = oracle.encode(imagegen.make("g1", w + 1, h, c, 1), w + 1, h, c, 0)
        pdata, poffsets, ppsizes = packed_device(files + [other])
        for name, buf, view in windows(n + 1, h, w, d):
            v = view[:n]
            guard = buf.clone()
            _, status = gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d, out=v)
            status = status.cpu().numpy()
            assert [s == 0 for s in status] == [e is not None for e in expect], (name, status)
            check_pixels_and_guard(buf, guard, v, expect, (name, w, h, c, d))
            buf.copy_(guard)
            _, status = gpu.decode_packed_device(pdata, poffsets, ppsizes, w, h, c, d, out=view,
                                                 max_file_size=max(len(f) for f in files + [other]))
            status = status.cpu().numpy()
            assert status[-1] == 100 and [s == 0 for s in status[:-1]] == [e is not None for e in expect], (name, status)
            check_pixels_and_guard(buf, guard, view, expect + [None], (name, "packed", w, h, c, d))


def check_pixels_and_guard(buf, guard, view, expect, what):
    """the view's images equal `expect` (None: the file failed, its pixels keep the guard), every other byte of buf is the guard"""
    import torch
    exp_buf = guard.clone()
    exp_view = exp_buf.as_strided(view.shape, view.stride(), view.storage_offset())
    for i, e in enumerate(expect):
        if e is not None:
            exp_view[i].copy_(torch.from_numpy(e.reshape(view.shape[1:])).cuda())
    assert torch.equal(buf, exp_buf), what


def test_round_trip_nchw_full_size(gpu):
    """256 x 3 x 1080 x 1920 NCHW -> planar encode -> decode_packed_device into NCHW: the input comes back, no host copy"""
    import torch
    n, c, h, w = 256, 3, 1080, 1920
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (torch.randint(0, 5, (n, c, h, w), generator=g, device="cuda", dtype=torch.uint8) * 50)
    x[:, :, ::7] = 17
    out, sizes = gpu.encode_batch_device(x.permute(0, 2, 3, 1))
    offsets = torch.arange(n, device="cuda", dtype=torch.int64) * out.stride(0)
    y = torch.empty_like(x)
    _, status = gpu.decode_packed_device(out.view(-1), offsets, sizes, w, h, c, c, out=y.permute(0, 2, 3, 1))
    assert int(status.abs().sum()) == 0
    assert torch.equal(x, y)
    del x, y, out


def test_strided_calls_reject_bad_layouts(gpu, oracle):
    """overlapping decode outputs, chan_stride 0 with pixel_stride 1, pixel_stride != chans for interleaved input:
    FPNGB_ERR_INVALID_ARG and nothing written"""
    import torch
    from fpng_b200._lib import lib
    L = lib()
    w, h, c, n = 40, 6, 3, 2
    src = torch.from_numpy(images("g1", n, w, h, 4, 1)).cuda()
    cap = (gpu.max_encoded_size(w, h, c) + 15) // 16 * 16
    out = torch.full((n, cap), GUARD, dtype=torch.uint8, device="cuda")
    sizes = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    enc = lambda *st: L.fpngb_encode_batch_device_strided(src.data_ptr(), *st, n, w, h, c, 0, out.data_ptr(), cap, sizes.data_ptr(), s)
    assert enc(h * w * 4, w * 4, 4, 1) == 1                                  # RGB view of RGBA pixels
    assert enc(h * w, w, 1, 0) == 1                                          # planar, chan_stride 0
    assert enc(h * w * 3, w * 3, 2, 1) == 1
    assert enc(h * w * 3, 1 << 33, 3, 1) == 1                                # row pitch beyond 32 bits
    torch.cuda.synchronize()
    assert bool((out == GUARD).all()) and bool((sizes == 7).all())
    # accepted: overlapping planes (plane k = plane 0 shifted down by k rows) of one broadcast image, all inside `rows`
    rows = torch.from_numpy(np.ascontiguousarray(imagegen.make("g1", w, h + c - 1, 3, 3)[..., 0]).reshape(-1)).cuda()
    assert L.fpngb_encode_batch_device_strided(rows.data_ptr(), 0, w, 1, w, n, w, h, c, 0, out.data_ptr(), cap, sizes.data_ptr(), s) == 0
    host = rows.cpu().numpy().reshape(h + c - 1, w)
    img = np.stack([host[k:k + h] for k in range(c)], axis=2)
    assert files_of(out, sizes) == [oracle.encode(np.ascontiguousarray(img), w, h, c, 0)] * n

    files = [oracle.encode(imagegen.make("g1", w, h, c, i), w, h, c, 0) for i in range(n)]
    t, stride, fsz, ofs, lens, *_ = gpu.pack_files_for_device(files, device="cuda")
    pix = torch.full((n * h * w * 4 + 64,), GUARD, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 9, dtype=torch.int32, device="cuda")
    data, offsets, psz = packed_device(files)
    fsz_a, ofs_a, lens_a = (np.ascontiguousarray(a, dtype=np.uint32) for a in (fsz, ofs, lens))
    for d in (3, 4):
        for st in ((h * w * d, w * d - 1, d, 1),                             # rows overlap
                   (h * w * d - 1, w * d, d, 1),                             # images overlap
                   (h * w * d, w, 1, 0),                                     # planar, chan_stride 0
                   (h * w * d, w * d, 1, 1),                                 # planar planes overlap
                   (h * w * d, w * 4, 4, 1) if d == 3 else (h * w * d, w * d, 3, 1)):   # pixel stride != chans
            rc = L.fpngb_decode_batch_device_strided(t.data_ptr(), stride, fsz_a.ctypes.data_as(C.c_void_p), ofs_a.ctypes.data_as(C.c_void_p),
                                                     lens_a.ctypes.data_as(C.c_void_p), n, w, h, c, d, pix.data_ptr(), *st,
                                                     status.data_ptr(), s)
            assert rc == 1, (d, st)
            rc = L.fpngb_decode_packed_device_strided(data.data_ptr(), offsets.data_ptr(), psz.data_ptr(), n, 1 << 20, w, h, c, d,
                                                      pix.data_ptr(), *st, status.data_ptr(), s)
            assert rc == 1, (d, st)
    torch.cuda.synchronize()
    assert bool((pix == GUARD).all()) and bool((status == 9).all())
