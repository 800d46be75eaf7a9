"""GPU tests of fpngb_decode_packed_ragged_device: packed device files of mixed widths, heights and channel counts decoded in
one call, the pixels placed back to back.  Pixels and statuses must equal the oracle's file by file, the output offsets a
numpy restatement of the placement rule, the walk rows get_info_batch_device's, and each shape group the bytes
decode_packed_device writes for that group alone.  Bytes of the output outside the decoded files must stay untouched."""
import numpy as np
import pytest

import imagegen
from test_decode_device_gpu import L, flip_corpus, surgery_corpus, to_device  # noqa: F401  (L: fixture)
from test_decoder_model_cpu import model_repairs

pytestmark = pytest.mark.gpu

INVALID_ARG, TOO_LARGE, SHAPE_MISMATCH, OUT_OF_SPACE = 2, 6, 100, 101
GUARD = 0xA5


def pack_at(files, rs, aligned16):
    """host buffer with the files in order, each at a 16-byte boundary (aligned16) or at a random multiple of 4; returns
    (buffer, offsets).  The buffer ends exactly at the end of the last file."""
    offs, at = [], 0
    for f in files:
        at = (at + 15) // 16 * 16 + (0 if aligned16 else 4 * int(rs.randint(0, 4)))
        offs.append(at)
        at += len(f)
    buf = np.zeros(at, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(bytes(f), np.uint8)
    return buf, offs


def placement(gpu, files, offs, base_bytes, d, max_file_size, max_w, max_h, out_cap):
    """numpy restatement of steps 1-4: (pre-status per file, 0 = decoded; out_offsets [n + 1] as uint64)"""
    pre, offsets, at = [], [], 0
    for f, o in zip(files, offs):
        size = len(f)
        info = gpu.get_info_ex(f) if size else (INVALID_ARG, 0, 0, 0, 0, 0)
        st, w, h = info[0], info[1], info[2]
        if not size or size > max_file_size or o % 4 or o + size > base_bytes:
            st = INVALID_ARG
        elif st == 0 and (w > max_w or h > max_h):
            st = SHAPE_MISMATCH
        elif st == 0 and w * h * d > 0xFFFFFFFF:
            st = TOO_LARGE
        offsets.append(at)
        if st == 0:
            take = (w * h * d + 15) // 16 * 16
            if at + take > out_cap:
                st = OUT_OF_SPACE
            at += take
        pre.append(st)
    total = at | ((1 << 63) if at > out_cap else 0)
    return pre, np.array(offsets + [total], np.uint64)


def run(gpu, data, offsets, sizes, d, out_cap, bounds, guard_tail=64):
    """the ragged call into a guard-filled output of out_cap (+ guard_tail) bytes; returns host copies of
    (out, out_offsets as uint64, info, status)"""
    import torch
    out = torch.full((out_cap + guard_tail,), GUARD, dtype=torch.uint8, device="cuda")
    mfs, mw, mh = bounds
    _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out[:out_cap], max_file_size=mfs, max_w=mw,
                                                      max_h=mh)
    torch.cuda.synchronize()
    return out.cpu().numpy(), oo.cpu().numpy().view(np.uint64), info.cpu().numpy(), st.cpu().numpy()


def check_call(gpu, oracle, files, offs, buf, d, bounds, out_cap=None):
    """one ragged call against the oracle, the placement model and get_info_batch_device; returns (statuses, out, offsets)"""
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    pre, want_offs = placement(gpu, files, offs, len(buf), d, *bounds, out_cap=1 << 62)
    total = int(want_offs[-1])
    if out_cap is None:
        out_cap = total
    pre, want_offs = placement(gpu, files, offs, len(buf), d, *bounds, out_cap=out_cap)
    out, oo, info, st = run(gpu, data, offsets, sizes, d, out_cap, bounds)
    assert np.array_equal(oo, want_offs), (d, oo[-3:], want_offs[-3:])
    walk = gpu.get_info_batch_device(data, offsets, sizes).cpu().numpy()
    written = np.zeros(out.size, bool)
    for i, f in enumerate(files):
        if pre[i] == INVALID_ARG:
            assert tuple(info[i]) == (INVALID_ARG, 0, 0, 0, 0, 0), (i, info[i])
        else:
            assert np.array_equal(info[i], walk[i]), (i, info[i], walk[i])
        est, epx = oracle.decode(f, d)[:2] if pre[i] == 0 else (pre[i], None)
        assert st[i] == est, (d, i, st[i], est, pre[i])
        if est == 0:
            o = int(oo[i])
            assert np.array_equal(out[o:o + epx.size], epx), (d, i)
            written[o:o + epx.size] = True
    assert (out[~written] == GUARD).all(), (d, np.flatnonzero(~written & (out != GUARD))[:8])
    return st, out, oo


def mixed_corpus(gpu, oracle, rs):
    import torch
    files = []
    shapes = [(1, 5), (2, 3), (15, 7), (16, 4), (17, 9), (687, 41), (1920, 12), (64, 1), (300, 20)]
    for j, (w, h) in enumerate(shapes):
        for c in (3, 4):
            for flags, kind in ((0, "g1"), (1, "g0"), (2, "runs"), (1, "g2")):
                files.append(oracle.encode(imagegen.make(kind, w, h, c, 40 + j), w, h, c, flags))
    # GPU-written files (encode_batch_device, 1-pass)
    for (w, h, c) in ((640, 48, 3), (17, 33, 4), (1920, 8, 4)):
        imgs = np.stack([imagegen.make(k, w, h, c, 5) for k in ("g1", "g0")])
        out, sizes = gpu.encode_batch_device(torch.from_numpy(imgs).cuda())
        out, sizes = out.cpu().numpy(), sizes.cpu().numpy()
        files += [out[i, :sizes[i]].tobytes() for i in range(len(imgs))]
    order = rs.permutation(len(files))
    return [files[i] for i in order]


def bounds_of(gpu, files):
    infos = [gpu.get_info_ex(f) for f in files if f]
    ok = [i for i in infos if i[0] == 0]
    return max(len(f) for f in files), max(i[1] for i in ok), max(i[2] for i in ok)


# ---- 1. mixed-shape parity -----------------------------------------------------------------------------------------------
def test_mixed_shape_parity(gpu, oracle):
    rs = np.random.RandomState(3)
    files = mixed_corpus(gpu, oracle, rs)
    # container and stream failures among them
    bad = bytearray(files[5]); bad[17] ^= 1
    files += [bytes(bad), files[6][:40], files[7][:-20], b"\0" + files[8][1:]]
    bounds = bounds_of(gpu, files)
    seen = set()
    for aligned16 in (True, False):
        buf, offs = pack_at(files, rs, aligned16)
        for d in (3, 4):
            st, _, _ = check_call(gpu, oracle, files, offs, buf, d, bounds)
            seen.update(st.tolist())
    assert {0, 3, 4, 7} <= seen, seen


def test_reference_written_files(gpu, oracle):
    """reference-written files (the oracle's encoder is byte-identical to the reference's: test_oracle_cpu / refreplay), of
    several shapes in one call"""
    rs = np.random.RandomState(4)
    files = [oracle.encode(imagegen.make(k, w, h, c, 11), w, h, c, flags)
             for (k, w, h, c) in (("g1", 640, 200, 3), ("g1", 640, 200, 4), ("g0", 1024, 128, 4), ("runs", 800, 60, 3), ("g2", 100, 40, 4))
             for flags in (0, 1, 2)]
    files = [files[i] for i in rs.permutation(len(files))]
    buf, offs = pack_at(files, rs, False)
    for d in (3, 4):
        st, _, _ = check_call(gpu, oracle, files, offs, buf, d, bounds_of(gpu, files))
        assert (st == 0).all()


# ---- 2. the same bytes as the uniform call, repairs ------------------------------------------------------------------------
@pytest.mark.parametrize("pre_roll", [256, 0])
def test_same_bytes_as_uniform_call(gpu, L, oracle, pre_roll):  # noqa: F811
    import torch
    rs = np.random.RandomState(9)
    files = []
    for (k, w, h, c, flags) in (("u128", 1024, 160, 3, 1), ("u16", 1024, 160, 4, 1), ("g1", 97, 13, 4, 0), ("g1", 97, 13, 4, 1),
                                ("g0", 200, 20, 3, 0), ("runs", 200, 20, 3, 1), ("g2", 31, 9, 4, 2), ("g1", 1024, 160, 3, 0)):
        files += [oracle.encode(imagegen.make(k, w, h, c, s), w, h, c, flags) for s in range(2)]
    bad = bytearray(files[4]); bad[len(bad) // 2] ^= 8; files.append(bytes(bad))
    files = [files[i] for i in rs.permutation(len(files))]
    want_repairs = sum(model_repairs(f, pre_roll) for f in files)
    assert want_repairs > 0
    buf, offs = pack_at(files, rs, True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    infos = [gpu.get_info_ex(f) for f in files]
    groups = {}
    for i, inf in enumerate(infos):
        groups.setdefault(inf[1:4], []).append(i)
    bounds = bounds_of(gpu, files)
    assert L.fpngb_debug_decode_preroll(pre_roll) == 0
    for d in (3, 4):
        L.fpngb_debug_decode_repairs(1)
        out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, max_file_size=bounds[0], max_w=bounds[1],
                                                            max_h=bounds[2])
        torch.cuda.synchronize()
        assert int(L.fpngb_debug_decode_repairs(1)) == want_repairs, d
        views = gpu.ragged_views(out, oo, info, st, d)
        st = st.cpu().numpy()
        for (w, h, c), idx in groups.items():
            sub = offsets[idx]
            px, ust = gpu.decode_packed_device(data, sub, sizes[idx], w, h, c, d, max_file_size=bounds[0])
            ust = ust.cpu().numpy()
            assert np.array_equal(ust, st[idx]), ((w, h, c), d)
            for k, i in enumerate(idx):
                if ust[k] == 0:
                    assert torch.equal(views[i], px[k]), ((w, h, c), d, i)
                else:
                    assert views[i] is None


# ---- 3. statuses and guards ------------------------------------------------------------------------------------------------
def test_statuses_and_guards(gpu, oracle):
    rs = np.random.RandomState(12)
    enc = lambda k, w, h, c, s, fl=0: oracle.encode(imagegen.make(k, w, h, c, s), w, h, c, fl)  # noqa: E731
    good = [enc("g1", 64, 16, 4, 1), enc("g0", 33, 7, 3, 2), enc("g1", 120, 30, 3, 3, 1), enc("runs", 48, 48, 4, 4)]
    wide, tall = enc("g1", 200, 8, 3, 5), enc("g1", 20, 90, 4, 6)
    max_size = max(len(f) for f in good + [wide, tall])
    big = good[0] + bytes(max_size)                                              # valid, larger than max_file_size
    damaged = [bytearray(good[k % 4]) for k in range(6)]
    for k, b in enumerate(damaged):
        b[int(rs.randint(60, len(b)))] ^= 1 << int(rs.randint(0, 8))
    files = good + [wide, tall, b"", big, good[1][:-9]] + [bytes(b) for b in damaged] + good
    corpus = flip_corpus(oracle, rs)[::40] + surgery_corpus(oracle)[::3]
    files += corpus
    buf, offs = pack_at(files, rs, True)
    # at the end: a copy 2 bytes past a 4-byte boundary, and a 4-aligned file that runs past the buffer's end
    mis_at = (len(buf) + 15) // 16 * 16 + 2
    buf = np.concatenate([buf, np.zeros(mis_at - len(buf), np.uint8), np.frombuffer(good[2], np.uint8)])
    files += [good[2], good[3]]
    offs += [mis_at, (len(buf) - len(good[3]) // 2) // 4 * 4]
    bounds = (max_size, 150, 60)
    for d in (3, 4):
        st, out, oo = check_call(gpu, oracle, files, offs, buf, d, bounds)
        assert st[4] == SHAPE_MISMATCH and st[5] == SHAPE_MISMATCH and st[6] == INVALID_ARG and st[7] == INVALID_ARG
        assert st[-2] == INVALID_ARG and st[-1] == INVALID_ARG
        assert {0, 1, 3, 4, 7} <= set(st.tolist()), set(st.tolist())
        total = int(oo[-1])
        # out_cap too small by one byte, then by several files: the placed prefix fits, bit 63 and the total
        placed = [i for i in range(len(files)) if oo[i + 1] != oo[i]]
        for cut in (1, int(total - oo[placed[len(placed) // 2]])):
            cap = total - cut
            st2, _, oo2 = check_call(gpu, oracle, files, offs, buf, d, bounds, out_cap=cap)
            assert int(oo2[-1]) == total | (1 << 63)
            assert np.array_equal(oo2[:-1], oo[:-1])
            for i in placed:
                fits = int(oo[i + 1]) <= cap
                assert (st2[i] == OUT_OF_SPACE) == (not fits), (cut, i, st2[i])
                if fits:
                    assert st2[i] == st[i]


def test_dimensions_too_large_and_rejected_calls(gpu, oracle):
    import torch
    from test_container_cpu import _chunk, _split
    png = oracle.encode(imagegen.make("g1", 64, 16, 4, 1), 64, 16, 4, 0)
    sig, ch = _split(png)
    ihdr = bytearray(ch[0][1]); ihdr[0:4] = (1 << 15).to_bytes(4, "big"); ihdr[4:8] = (1 << 15).to_bytes(4, "big")
    huge = sig + _chunk(b"IHDR", bytes(ihdr)) + ch[1][2] + ch[2][2] + ch[3][2]     # 2^30 pixels: 2^32 bytes at 4 channels
    files = [png, huge]
    buf, offs = pack_at(files, np.random.RandomState(0), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    for d, want in ((3, OUT_OF_SPACE), (4, TOO_LARGE)):
        out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, max_file_size=len(huge), max_w=1 << 15, max_h=1 << 15,
                                                            out=torch.empty(4096, dtype=torch.uint8, device="cuda"))
        st = st.cpu().numpy()
        assert st[0] == 0 and st[1] == want, (d, st)
    # rejected calls enqueue nothing and write nothing
    from fpng_b200._lib import lib
    out = torch.full((4096,), GUARD, dtype=torch.uint8, device="cuda")
    oo = torch.full((3,), -7, dtype=torch.int64, device="cuda"); info = torch.full((2, 6), -7, dtype=torch.int32, device="cuda")
    st = torch.full((2,), -7, dtype=torch.int32, device="cuda")
    base = (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr())
    tail = lambda o=out.data_ptr(): (o, 4096, oo.data_ptr(), info.data_ptr(), st.data_ptr(), None)  # noqa: E731
    for args, rc in (((2, 5000, 64, 16, 5), 1), ((2, 5000, 64, 16, 2), 1), ((0, 5000, 64, 16, 4), 1), ((65536, 5000, 64, 16, 4), 1),
                     ((2, 0, 64, 16, 4), 1), ((2, 5000, 0, 16, 4), 1), ((2, 5000, 64, 0, 4), 1), ((2, 5000, (1 << 24) + 1, 16, 4), 1),
                     ((2, 5000, 64, (1 << 24) + 1, 4), 1)):
        assert lib().fpngb_decode_packed_ragged_device(*base, *args, *tail()) == rc, args
    assert lib().fpngb_decode_packed_ragged_device(*base, 2, 5000, 64, 16, 4, *tail(out.data_ptr() + 8)) == 5
    assert lib().fpngb_decode_packed_ragged_device(data.data_ptr() + 2, *base[1:], 2, 5000, 64, 16, 4, *tail()) == 5
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == GUARD).all() and (oo.cpu().numpy() == -7).all()
    assert (info.cpu().numpy() == -7).all() and (st.cpu().numpy() == -7).all()


# ---- 4. a uniform batch through the ragged call ----------------------------------------------------------------------------
def test_uniform_round_trip_full_size(gpu):
    import torch
    from fpng_b200 import dist
    w, h, c = 1920, 1080, 3
    imgs = np.stack([imagegen.make("g1", w, h, c, i) for i in range(8)])
    dev = torch.from_numpy(imgs).cuda()
    out, sizes = gpu.encode_batch_device(dev)
    flat, offsets = dist.compact(out, sizes)
    px, oo, info, st = gpu.decode_packed_ragged_device(flat, offsets, sizes, c)
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == 0).all()
    assert px.numel() == len(imgs) * w * h * c and torch.equal(px.view(len(imgs), h, w, c), dev)
    assert [v.shape for v in gpu.ragged_views(px, oo, info, st, c)] == [(h, w, c)] * len(imgs)


# ---- 5. no host synchronisation --------------------------------------------------------------------------------------------
def test_no_host_synchronisation(gpu, oracle):
    import torch
    files = [oracle.encode(imagegen.make("g1", w, h, c, i), w, h, c, 0) for i, (w, h, c) in enumerate(((512, 64, 4), (100, 30, 3), (7, 90, 4)))]
    buf, offs = pack_at(files, np.random.RandomState(1), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=512, max_h=90)
    out = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out, **bounds)     # workspace reserved before the timed call
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)                                           # ~0.5 s of GPU time in front of the call
        _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out, **bounds)
        assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert (st.cpu().numpy() == 0).all()
    for i, v in enumerate(gpu.ragged_views(out, oo, info, st, 4)):
        assert np.array_equal(v.cpu().numpy().reshape(-1), oracle.decode(files[i], 4)[1]), i
