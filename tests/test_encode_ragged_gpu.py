"""GPU tests of fpngb_encode_ragged_device: device images of mixed widths, heights, channel counts and layouts encoded in one
call into one packed buffer.  Every file must equal the oracle's encode of that image and, per shape group, what
encode_batch_device writes for the group alone; the slot offsets must equal a numpy restatement of the slot rule, and no byte
past the total may be written.  The result must round-trip through decode_packed_ragged_device, also after
compact_packed_device."""
import ctypes as C

import numpy as np
import pytest

import imagegen
from test_trained_tables_cpu import load_tables

pytestmark = pytest.mark.gpu

INVALID_ARG, TOO_SMALL, ALIGNMENT = 1, 2, 5
GUARD = 0xA5
WIDTHS = [1, 2, 15, 16, 17, 511, 512, 513, 687, 1920]
HEIGHTS = list(range(1, 12)) + [40, 41, 1080]
FLAGS = (0, 1, 2)                                  # 0, FPNG_ENCODE_SLOWER, FPNG_FORCE_UNCOMPRESSED


@pytest.fixture
def rows_per_warp(request):
    """Forces the scanlines-per-warp shape of the pack kernel (0 = automatic), so that small images take the multi-scanline
    sequence too."""
    from fpng_b200 import _lib
    _lib.lib().fpngb_debug_rows_per_warp(request.param)
    yield request.param
    _lib.lib().fpngb_debug_rows_per_warp(0)


def shapes_mix():
    """every width and every height at least once per channel count, (h, w, c); the 1080-row image is 687 wide"""
    out = []
    for c in (3, 4):
        for k, w in enumerate(WIDTHS):
            out.append((HEIGHTS[(k + 3 * c) % 13], w, c))
        for h in HEIGHTS:
            out.append((h, 687 if h == 1080 else 17 + h, c))
    return out


def host_images(shapes, kind="g1", seed=0):
    return [imagegen.make(kind, w, h, c, seed + i).reshape(h, w, c) for i, (h, w, c) in enumerate(shapes)]


def files_of(out, offsets, sizes):
    out = out.cpu().numpy()
    offs = offsets.cpu().numpy()
    sz = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return [out[offs[i]:offs[i] + sz[i]].tobytes() for i in range(len(sz))]


def launches(gpu, fn):
    import torch
    torch.cuda.synchronize()
    before = gpu.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return gpu.launch_count() - before, r


def check_oracle(oracle, hosts, files, flags, what=""):
    for i, (img, f) in enumerate(zip(hosts, files)):
        h, w, c = img.shape
        assert f == oracle.encode(np.ascontiguousarray(img), w, h, c, flags), (what, i, h, w, c, flags)


# ---- 1. parity with the oracle ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows_per_warp", [1, 5], indirect=True)
@pytest.mark.parametrize("flags", FLAGS)
def test_parity_mixed_shapes(gpu, oracle, flags, rows_per_warp):
    import torch
    shapes = shapes_mix()
    hosts = host_images(shapes, "g1", 100 * flags)
    dev = [torch.from_numpy(x).cuda() for x in hosts]
    files = files_of(*gpu.encode_ragged_device(dev, flags))
    check_oracle(oracle, hosts, files, flags, "mix")


@pytest.mark.parametrize("flags", (0, 1))
def test_parity_stored_fallback(gpu, oracle, flags):
    """random bytes: every file falls back to stored blocks"""
    import torch
    shapes = [(9, 687, 3), (4, 1920, 4), (3, 16, 3), (41, 513, 4), (1, 1, 3)]
    hosts = host_images(shapes, "g2", 3)
    files = files_of(*gpu.encode_ragged_device([torch.from_numpy(x).cuda() for x in hosts], flags))
    check_oracle(oracle, hosts, files, flags, "stored")
    assert all(len(f) >= (w * c + 1) * h for f, (h, w, c) in zip(files, shapes)), "expected the stored-block fallback"


# ---- 2. same bytes as the uniform call per shape group ----------------------------------------------------------------------
@pytest.mark.parametrize("flags", FLAGS)
def test_same_bytes_as_uniform_call(gpu, flags):
    import torch
    groups = [(5, 687, 3, 3), (4, 64, 4, 2), (40, 17, 3, 4), (2, 1920, 4, 2)]          # (h, w, c, count)
    imgs = [torch.from_numpy(np.stack(host_images([(h, w, c)] * k, "runs", 10 * gi))).cuda() for gi, (h, w, c, k) in enumerate(groups)]
    order = [(g, j) for j in range(4) for g in range(len(groups)) if j < groups[g][3]]    # groups interleaved
    files = files_of(*gpu.encode_ragged_device([imgs[g][j] for g, j in order], flags))
    for g, batch in enumerate(imgs):
        out, sizes = gpu.encode_batch_device(batch, flags)
        sz = sizes.cpu().numpy()
        uni = [out[i, :sz[i]].cpu().numpy().tobytes() for i in range(batch.shape[0])]
        got = [files[k] for k, (gg, j) in enumerate(order) if gg == g]
        assert got == uni, groups[g]


# ---- 3. layouts: all six (chans x loader) classes, launch count ---------------------------------------------------------------
def layout_mix(torch):
    """(device view, host pixels) pairs covering staged, direct and planar loaders for 3 and 4 channels"""
    views = []
    for c in (3, 4):
        w, h = 80, 7
        canvas_host = imagegen.make("g1", w + 16, h + 2, c, c).reshape(h + 2, w + 16, c)
        canvas = torch.from_numpy(canvas_host).cuda()
        for x0 in range(16):                                                   # crops: x0 = 0 (c=4) is staged, the rest direct
            views.append((canvas[1:1 + h, x0:x0 + w], canvas_host[1:1 + h, x0:x0 + w]))
        src = imagegen.make("g1", 33, 9, c, 7 + c).reshape(9, 33, c)
        chw = torch.from_numpy(np.ascontiguousarray(src.transpose(2, 0, 1))).cuda()
        views.append((chw.permute(1, 2, 0), src))                            # NCHW permute: planar
        cs = 9 * 33 + 3                                                        # odd plane stride
        flat = torch.full((c * cs + 16,), 0x5A, dtype=torch.uint8, device="cuda")
        odd = flat.as_strided((9, 33, c), (33, 1, cs), 1)
        odd.copy_(torch.from_numpy(src).cuda())
        views.append((odd, src))
        tight = torch.from_numpy(imagegen.make("runs", 64, 5, c, 1).reshape(5, 64, c)).cuda()
        views.append((tight, tight.cpu().numpy()))                             # 16-byte aligned rows: staged
        views.append((tight, tight.cpu().numpy()))                             # the same tensor twice
    return views


@pytest.mark.parametrize("flags", (0, 1))
def test_layouts_in_one_call(gpu, oracle, flags):
    import torch
    views = layout_mix(torch)
    # classes: (c, loader) from the rule of the uniform launch
    classes = set()
    for v, _ in views:
        h, w, c = v.shape
        st = v.stride()
        planar = st[1] == 1 and c > 1
        staged = not planar and v.data_ptr() % 16 == 0 and (st[0] % 16 == 0 or h == 1) and (w * c) % 16 == 0
        classes.add((c, "planar" if planar else "staged" if staged else "direct"))
    assert len(classes) == 6, classes
    k, res = launches(gpu, lambda: gpu.encode_ragged_device([v for v, _ in views], flags))
    files = files_of(*res)
    check_oracle(oracle, [h for _, h in views], files, flags, "layouts")
    # documented launch count: per non-empty class scan + pack (+ hist), per-image kernels offsets, Adler, row-CRC, stored CRC
    # (+ Huffman build)
    two_pass = flags == 1
    assert k == 6 * (3 if two_pass else 2) + 4 + (1 if two_pass else 0), k


def test_profile_slots(gpu):
    import torch
    from fpng_b200 import _lib
    L = _lib.lib()
    imgs = [torch.from_numpy(x).cuda() for x in host_images([(30, 100, 3), (20, 64, 4)])]
    L.fpngb_profile_enable(1)
    try:
        gpu.encode_ragged_device(imgs, 1)
        ms = (C.c_float * 9)()
        calls = L.fpngb_profile_read(ms, 9)
    finally:
        L.fpngb_profile_enable(0)
    # slots: hist, huffman, scan, offsets, (single-pass encoder, its finish), pack, adler, crc
    assert calls == 1 and all(ms[i] > 0 for i in (0, 1, 2, 3, 6, 7, 8)) and ms[4] == ms[5] == 0, list(ms)


# ---- 4. slots --------------------------------------------------------------------------------------------------------------
def test_slots_and_guard(gpu, oracle):
    import torch
    shapes = [(7, 13, 3), (1, 1, 4), (40, 687, 4), (11, 512, 3), (2, 1920, 3)]
    hosts = host_images(shapes)
    total = int(gpu.ragged_slot_offsets(shapes)[-1])
    want = np.zeros(len(shapes) + 1, np.int64)
    for i, (h, w, c) in enumerate(shapes):
        raw = (w * c + 1) * h
        stored = 58 + 6 + raw + 5 * ((raw + 65534) // 65535) + 16
        comp = ((58 + raw + 7) & ~7) + 16
        want[i + 1] = want[i] + (max(stored, comp) + 15) // 16 * 16
    assert total == want[-1]
    out = torch.full((total + 4096,), GUARD, dtype=torch.uint8, device="cuda")
    _, offsets, sizes = gpu.encode_ragged_device([torch.from_numpy(x).cuda() for x in hosts], 0, out=out)
    assert np.array_equal(offsets.cpu().numpy(), want)
    assert (out[total:].cpu().numpy() == GUARD).all(), "bytes past the total were written"
    check_oracle(oracle, hosts, files_of(out, offsets, sizes), 0, "slots")


# ---- 5. trained tables -----------------------------------------------------------------------------------------------------
def test_trained_tables(gpu, oracle):
    """RGB and RGBA images run the ragged kernels under the trained tables (for RGBA the one-pixel-match rule's instantiations)
    and equal the oracle running the same tables"""
    import torch
    tables = load_tables()
    try:
        for chans in (3, 4):
            t = tables[str(chans)]
            prefix = bytes.fromhex(t["prefix"])
            assert oracle.set_static_table(chans, prefix, t["bit_buf"], t["bit_buf_size"])
            gpu.set_static_table(chans, prefix, t["bit_buf"], t["bit_buf_size"])
        hosts, names = [], []
        for chans in (3, 4):
            sizes = np.array(tables[str(chans)]["sizes"], np.uint8)
            for (name, w, h, img) in imagegen.trained_table_images(chans, sizes):
                hosts.append(np.asarray(img).reshape(h, w, chans)); names.append((chans, name))
        files = files_of(*gpu.encode_ragged_device([torch.from_numpy(x).cuda() for x in hosts], 0))
        check_oracle(oracle, hosts, files, 0, "trained")
    finally:
        for chans in (3, 4):
            gpu.set_static_table(chans)
            oracle.set_static_table(chans)


# ---- 6. rejections ---------------------------------------------------------------------------------------------------------
def test_rejections(gpu):
    import torch
    from fpng_b200 import _lib
    L = _lib.lib()
    img = torch.from_numpy(imagegen.make("g1", 20, 6, 3, 1).reshape(6, 20, 3)).cuda()
    total = int(gpu.ragged_slot_offsets([(6, 20, 3)])[-1])
    out = torch.full((total + 64,), GUARD, dtype=torch.uint8, device="cuda")
    offsets = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def call(n=1, ptrs=None, dims=None, strides=None, out_ptr=None, cap=None):
        p = np.array([img.data_ptr()] if ptrs is None else ptrs, np.uint64)
        d = np.array([[20, 6, 3]] if dims is None else dims, np.uint32)
        st = None if strides is None else np.array(strides, np.uint64)
        return L.fpngb_encode_ragged_device(n, p.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                            None if st is None else st.ctypes.data_as(C.c_void_p), 0,
                                            out.data_ptr() if out_ptr is None else out_ptr, total if cap is None else cap,
                                            offsets.data_ptr(), sizes.data_ptr(), s)

    cases = [
        (INVALID_ARG, dict(n=0)),
        (INVALID_ARG, dict(n=65536, ptrs=[img.data_ptr()] * 65536, dims=[[20, 6, 3]] * 65536)),
        (INVALID_ARG, dict(ptrs=[0])),
        (INVALID_ARG, dict(dims=[[0, 6, 3]])),
        (INVALID_ARG, dict(dims=[[20, 6, 2]])),
        (INVALID_ARG, dict(strides=[[60, 4, 1]])),                               # an RGB view of RGBA pixels
        (TOO_SMALL, dict(cap=total - 1)),
        (ALIGNMENT, dict(out_ptr=out.data_ptr() + 4)),
    ]
    for want, kw in cases:
        k, rc = launches(gpu, lambda: call(**kw))
        assert rc == want and k == 0, (kw.keys(), rc, k)
    assert (out.cpu().numpy() == GUARD).all() and (offsets.cpu().numpy() == -7).all() and (sizes.cpu().numpy() == -7).all()
    assert L.fpngb_encode_ragged_device(1, None, None, None, 0, out.data_ptr(), total, offsets.data_ptr(), sizes.data_ptr(), s) == INVALID_ARG
    assert call() == 0                                                          # the same arguments otherwise pass


# ---- 7. round trip, compaction -------------------------------------------------------------------------------------------
def test_round_trip_and_compaction(gpu):
    import torch
    shapes = [(h, w, c) for (h, w, c) in shapes_mix() if h * w < 200000][:30]
    hosts = host_images(shapes, "g1", 5)
    data, offsets, sizes = gpu.encode_ragged_device([torch.from_numpy(x).cuda() for x in hosts], 0)

    def decoded(d, o, s):
        res = []
        for c in (3, 4):
            out, oo, info, st = gpu.decode_packed_ragged_device(d, o, s, c)
            assert (st.cpu().numpy() == 0).all()
            res.append(gpu.ragged_views(out, oo, info, st, c))
        return res

    def check(views3, views4):
        for i, x in enumerate(hosts):
            v = (views3 if x.shape[2] == 3 else views4)[i]
            assert np.array_equal(v.cpu().numpy(), x), i

    check(*decoded(data, offsets, sizes))
    cdata, coffs = gpu.compact_packed_device(data, offsets, sizes)
    sz = sizes.cpu().numpy().astype(np.int64)
    want = np.concatenate([[0], np.cumsum((sz + 15) // 16 * 16)])
    assert np.array_equal(coffs.cpu().numpy(), want)
    assert want[-1] < int(offsets[-1])
    check(*decoded(cdata[:want[-1]], coffs, sizes))
    # dst_cap short: bit 63 of the total, the files that do not fit are not copied
    cut = int(want[len(want) // 2]) + 8
    small = torch.full((cut + 64,), GUARD, dtype=torch.uint8, device="cuda")
    _, coffs2 = gpu.compact_packed_device(data, offsets, sizes, out=small[:cut])
    o2 = coffs2.cpu().numpy().astype(np.uint64)
    assert o2[-1] == np.uint64(want[-1]) | np.uint64(1 << 63)
    host_small = small.cpu().numpy()
    assert (host_small[cut:] == GUARD).all()
    dh = data.cpu().numpy(); oh = offsets.cpu().numpy()
    fits = want[1:] <= cut                                                     # the copied files are a prefix
    first_out = int(np.argmin(fits))
    assert not fits[first_out] and fits[:first_out].all()
    for i in range(first_out):
        assert np.array_equal(host_small[want[i]:want[i] + sz[i]], dh[oh[i]:oh[i] + sz[i]]), i
    assert (host_small[want[first_out]:cut] == GUARD).all(), "a file that does not fit was copied"


# ---- 8. full size ----------------------------------------------------------------------------------------------------------
def test_full_size(gpu, oracle):
    import torch
    shapes = [(2160, 3840, 4), (1080, 1920, 3), (1012, 687, 3)]
    hosts = host_images(shapes, "g1", 9)
    files = files_of(*gpu.encode_ragged_device([torch.from_numpy(x).cuda() for x in hosts], 0))
    check_oracle(oracle, hosts, files, 0, "full")


# ---- 9. no host synchronisation --------------------------------------------------------------------------------------------
def test_no_host_synchronisation(gpu, oracle):
    import torch
    shapes = [(64, 512, 4), (30, 100, 3), (90, 7, 4)]
    hosts = host_images(shapes, "g1", 2)
    dev = [torch.from_numpy(x).cuda() for x in hosts]
    gpu.encode_ragged_device(dev, 0)                                          # workspace reserved before the timed calls
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)                                           # ~0.5 s of GPU time in front of the calls
        a = gpu.encode_ragged_device(dev, 0)
        b = gpu.encode_ragged_device(dev[::-1], 1)                            # the first call's staging is still in flight
        assert not s.query(), "a call waited for the stream"
    s.synchronize()
    check_oracle(oracle, hosts, files_of(*a), 0, "first")
    check_oracle(oracle, hosts[::-1], files_of(*b), 1, "second")


# ---- 10. trained tables on every RGBA loader -------------------------------------------------------------------------------
def test_trained_tables_mixed_layouts(gpu, oracle):
    """Under both trained tables (the RGBA one's one-pixel-match rule fires) a ragged call over RGB images and interleaved,
    cropped (direct loader) and planar RGBA views, of uint8 and of float32, writes the oracle's files with as many launches as
    the same call under the shipped tables: no image leaves the ragged pipeline."""
    import torch
    tables = load_tables()
    sizes = np.array(tables["4"]["sizes"], np.uint8)
    pal = [int(v) for v in np.argsort(sizes[:256], kind="stable")[:4]]
    rgba = [imagegen.short_runs(w, h, 4, 20 + i, pal) for i, (h, w) in enumerate([(24, 61), (9, 513), (5, 1030), (1, 16)])]
    hosts, u8, f32 = [], [], []
    for x in rgba + host_images([(9, 687, 3), (40, 17, 3)], "runs", 30):
        h, w, c = x.shape
        for layout in (("interleaved", "cropped", "planar") if c == 4 else ("interleaved",)):
            hosts.append(x)
            for dst, t in ((u8, torch.from_numpy(np.ascontiguousarray(x)).cuda()),
                           (f32, torch.from_numpy(np.ascontiguousarray(x)).cuda().float().div_(255))):
                if layout == "cropped":
                    canvas = torch.zeros((h, w + 3, c), dtype=t.dtype, device="cuda"); canvas[:, 3:] = t; t = canvas[:, 3:]
                elif layout == "planar":
                    t = t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
                dst.append(t)
    calls = {f"{name} {flags}": (lambda imgs=imgs, flags=flags, kw=kw: gpu.encode_ragged_device(imgs, flags, **kw))
             for name, imgs, kw in (("uint8", u8, {}), ("float32", f32, {"scale": 255.0})) for flags in (0, 1)}
    shipped = {name: launches(gpu, fn)[0] for name, fn in calls.items()}
    try:
        for chans in (3, 4):
            t = tables[str(chans)]
            prefix = bytes.fromhex(t["prefix"])
            assert oracle.set_static_table(chans, prefix, t["bit_buf"], t["bit_buf_size"])
            gpu.set_static_table(chans, prefix, t["bit_buf"], t["bit_buf_size"])
        for name, fn in calls.items():
            k, r = launches(gpu, fn)
            check_oracle(oracle, hosts, files_of(*r), int(name[-1]), name)
            assert k == shipped[name], (name, k, shipped[name])
    finally:
        for chans in (3, 4):
            gpu.set_static_table(chans)
            oracle.set_static_table(chans)
