"""GPU tests of the decode of files already in device memory: fpngb_get_info_batch_device (container_walk_kernel, the same
container walk as the host's fpngb_get_info_ex) and fpngb_decode_packed_device (walk + decode kernels over files packed back
to back, the layout of dist.compact and of the gather window).  Walk results must equal the host walk and the oracle's code,
statuses and pixels the oracle's decode, file by file."""
import numpy as np
import pytest

import imagegen
from test_container_cpu import _chunk, _split
from test_container_cpu import files as container_files

pytestmark = pytest.mark.gpu

INVALID_ARG, SHAPE_MISMATCH = 2, 100


def pack(files, odd=False):
    """host buffer with the files back to back: 16-byte aligned starts, or (odd) starts at an odd byte.  Returns
    (buffer, offsets); the buffer ends exactly at the end of the last file."""
    offs, at = [], 0
    for i, f in enumerate(files):
        at = (at + 15) // 16 * 16 + ((1 + 2 * (i % 4)) if odd else 0)
        offs.append(at)
        at += len(f)
    buf = np.zeros(at, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(bytes(f), np.uint8)
    return buf, offs


def to_device(buf, offs, sizes):
    import torch
    data = torch.from_numpy(np.array(buf, dtype=np.uint8)).cuda()
    offsets = torch.tensor(np.asarray(offs, np.int64)).cuda()
    sz = torch.from_numpy(np.asarray(sizes, np.uint32).view(np.int32).copy()).cuda()
    return data, offsets, sz


def packed_device(files, odd=False):
    buf, offs = pack(files, odd)
    return to_device(buf, offs, [len(f) for f in files])


@pytest.fixture
def L(gpu):
    from fpng_b200._lib import lib
    from test_decoder_model_cpu import K_PRE_ROLL
    L = lib()
    yield L
    L.fpngb_debug_decode_preroll(K_PRE_ROLL)                                 # the default


# ---- 1. walk parity ------------------------------------------------------------------------------------------------------
def flip_corpus(oracle, rs):
    out = []
    for png, w, h, c in container_files(oracle):
        out += [png[:k] for k in (7, 8, 20, 33, 40, 57, 58, len(png) - 13, len(png) - 12, len(png) - 1)]
        for _ in range(150):
            bad = bytearray(png)
            zone = int(rs.randint(0, 3))
            pos = int(rs.randint(0, min(100, len(bad)))) if zone == 0 else (len(bad) - 1 - int(rs.randint(0, min(24, len(bad)))) if zone == 1
                                                                             else int(rs.randint(0, len(bad))))
            bad[pos] ^= 1 << int(rs.randint(0, 8))
            out.append(bytes(bad))
        for _ in range(20):
            cut = int(rs.randint(8, len(png)))
            out.append(png[:cut] + bytes(rs.randint(0, 256, int(rs.randint(1, 40)), dtype=np.uint8)) + png[cut:])
    return out


def surgery_corpus(oracle):
    out = []
    for png, w, h, c in container_files(oracle):
        sig, ch = _split(png)
        ihdr, fdec, idat, iend = (r for _, _, r in ch)
        ihdr_body, idat_body = ch[0][1], ch[2][1]
        anc = _chunk(b"tEXt", b"Comment\0made by a test")
        out += [sig + ihdr + anc + fdec + idat + iend, sig + ihdr + fdec + idat + anc + iend, sig + ihdr + fdec + _chunk(b"zzZz", b"") + idat + iend,
                sig + ihdr + _chunk(b"PLTE", bytes(6)) + fdec + idat + iend, sig + ihdr + fdec + _chunk(b"tEXt", b"abc", good_crc=False) + idat + iend,
                sig + ihdr + fdec + idat + _chunk(b"IEND", b"", good_crc=False), sig + ihdr + fdec + _chunk(b"IDAT", idat_body, good_crc=False) + iend,
                sig + ihdr + fdec + fdec + idat + iend, sig + ihdr + idat + iend, sig + ihdr + idat + fdec + iend,
                sig + ihdr + _chunk(b"fdEC", bytes([82, 36, 147, 227, 1])) + idat + iend, sig + ihdr + _chunk(b"fdEC", bytes([82, 36, 147, 227])) + idat + iend,
                sig + ihdr + fdec + idat + idat + iend, sig + ihdr + fdec + _chunk(b"IDAT", idat_body[:6]) + iend,
                sig + ihdr + fdec + _chunk(b"IDAT", idat_body[:7]) + iend, sig + ihdr + fdec + iend, sig + ihdr + fdec + idat,
                sig + ihdr + iend + fdec + idat, png + b"\0" * 19, sig + ihdr + fdec + _chunk(b"tEX1", b"abc") + idat + iend,
                sig + ihdr + fdec + _chunk(b"`EXt", b"abc") + idat + iend, sig + ihdr + fdec + idat[:4] + b"IDAT",
                sig + ihdr + fdec + b"\xff\xff\xff\xff" + idat[4:] + iend, sig + ihdr + ihdr + fdec + idat + iend,
                sig + _chunk(b"IHDR", ihdr_body + b"\0") + fdec + idat + iend]

        def with_ihdr(**kw):
            b = bytearray(ihdr_body)
            for k, v in kw.items():
                if k == "w": b[0:4] = v.to_bytes(4, "big")
                elif k == "h": b[4:8] = v.to_bytes(4, "big")
                else: b[{"depth": 8, "ctype": 9, "comp": 10, "filt": 11, "lace": 12}[k]] = v
            return sig + _chunk(b"IHDR", bytes(b)) + fdec + idat + iend
        out += [with_ihdr(w=0), with_ihdr(h=0), with_ihdr(w=(1 << 24) + 1, h=1), with_ihdr(w=1 << 15, h=(1 << 15) + 1), with_ihdr(w=0xFFFFFFFF),
                with_ihdr(depth=16), with_ihdr(ctype=3), with_ihdr(ctype=2 if c == 4 else 6), with_ihdr(comp=1), with_ihdr(lace=1)]
    return out


def random_corpus(rs, trials=3000):
    """random chunk sequences (the generator of test_container_cpu's property test, another seed)"""
    sig = bytes([137, 80, 78, 71, 13, 10, 26, 10])

    def ihdr():
        plain = rs.rand() < 0.7
        w = int(rs.choice([1, 7, 640, 65535, 65536, 1 << 15] if plain else [0, 1 << 24, (1 << 24) + 1, 1 << 15]))
        h = int(rs.choice([1, 9, 480, 1 << 15] if plain else [0, (1 << 15) + 1, 1 << 24, 3]))
        depth = 8 if plain else int(rs.choice([8, 16, 1])); ctype = int(rs.choice([2, 6] if plain else [2, 6, 0, 3, 4]))
        flags = [int(rs.rand() < (0.0 if plain else 0.1)) for _ in range(3)]
        body = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([depth, ctype] + flags)
        if rs.rand() < 0.03:
            body += b"\0"
        return _chunk(b"IHDR", body, good_crc=rs.rand() > 0.03)

    def piece():
        k = rs.randint(0, 12)
        good = rs.rand() > 0.1
        if k <= 2:
            return _chunk(b"fdEC", bytes([82, 36, 147, 227, 0]) if rs.rand() > 0.15 else bytes(rs.randint(0, 256, rs.randint(0, 8), dtype=np.uint8)), good)
        if k <= 5:
            return _chunk(b"IDAT", bytes(rs.randint(0, 256, int(rs.choice([0, 6, 7, 8, 40, 200])), dtype=np.uint8)), good)
        if k <= 7:
            return _chunk(b"IEND", b"" if rs.rand() > 0.1 else b"x", good)
        if k == 8:
            return _chunk(bytes(rs.choice([b"tEXt", b"gAMA", b"zTXt", b"aaaa", b"prIv"])), bytes(rs.randint(0, 256, rs.randint(0, 20), dtype=np.uint8)), good)
        if k == 9:
            return _chunk(bytes(rs.choice([b"PLTE", b"ABCD", b"IDAU", b"Idat"])), bytes(rs.randint(0, 256, rs.randint(0, 20), dtype=np.uint8)), good)
        if k == 10:
            t = bytearray(b"tEXt"); t[rs.randint(0, 4)] = int(rs.choice([48, 64, 91, 96, 123, 0, 255]))
            return _chunk(bytes(t), b"abc", good)
        return bytes(rs.randint(0, 256, rs.randint(1, 16), dtype=np.uint8))

    out = []
    for _ in range(trials):
        f = (sig if rs.rand() > 0.03 else sig[:7] + b"\x0b") + ihdr()
        if rs.rand() < 0.6:
            f += _chunk(b"fdEC", bytes([82, 36, 147, 227, 0]))
        for _ in range(rs.randint(1, 5)):
            f += piece()
        if rs.rand() < 0.7:
            f += _chunk(b"IEND", b"")
        if rs.rand() < 0.15:
            f = f[: rs.randint(0, len(f) + 1)]
        if f:
            out.append(f)
    return out


def test_walk_parity(gpu, oracle):
    import torch
    rs = np.random.RandomState(31)
    png = oracle.encode(imagegen.make("g1", 64, 16, 3, 1), 64, 16, 3, 0)
    sig, ch = _split(png)
    big = sig + ch[0][2] + _chunk(b"zTXt", bytes(rs.randint(0, 256, 300 << 10, dtype=np.uint8))) + ch[1][2] + ch[2][2] + ch[3][2]
    big_bad = bytearray(big); big_bad[200 << 10] ^= 4                        # same chunk, CRC no longer matches
    corpus = flip_corpus(oracle, rs) + surgery_corpus(oracle) + random_corpus(rs) + [big, bytes(big_bad)]
    corpus.append(sig + ch[0][2] + ch[1][2] + b"\xff\xff\xff\xffIDAT" + ch[2][1][:20])   # length 0xFFFFFFFF in the buffer's last chunk
    want = [gpu.get_info_ex(f) for f in corpus]
    seen = set()
    for f, wt in zip(corpus, want):
        assert oracle.get_info(f)[0] == wt[0], f[:64]
        seen.add(wt[0])
    assert seen == {0, 1, 3, 4, 5, 7, 8}, seen
    assert want[-3][0] == 0 and want[-2][0] == 4 and want[-1][0] == 7
    for odd in (False, True):
        data, offsets, sizes = packed_device(corpus, odd)
        info = gpu.get_info_batch_device(data, offsets, sizes)
        torch.cuda.synchronize()
        info = info.cpu().numpy().view(np.uint32)
        for i, wt in enumerate(want):
            assert tuple(int(v) for v in info[i]) == tuple(wt), (odd, i, tuple(info[i]), wt, corpus[i][:64])
    # a size of 0 is an invalid argument, like fpng_decode_memory's empty buffer
    data, offsets, sizes = to_device(np.frombuffer(png, np.uint8), [0, 0], [0, len(png)])
    info = gpu.get_info_batch_device(data, offsets, sizes).cpu().numpy()
    assert info[0, 0] == INVALID_ARG and tuple(info[1]) == tuple(gpu.get_info_ex(png))


# ---- 2. decode parity on the packed layout -------------------------------------------------------------------------------
SHAPES = [(1, 1), (1, 9), (2, 2), (5, 3), (16, 2), (24, 1), (63, 3), (64, 3), (85, 2), (86, 2), (127, 5), (128, 4), (129, 6),
          (257, 33), (340, 5), (512, 64), (687, 41), (1000, 3), (2049, 2)]
KINDS = ["g0", "g1", "g2", "runs", "mut", "zero"]


def check_packed(gpu, oracle, files, w, h, c, d, expect=None, max_file_size=None):
    """decode_packed_device of `files` against the oracle (or `expect`: (status, pixels) per file), file by file; returns the
    statuses"""
    data, offsets, sizes = packed_device(files)
    out, status = gpu.decode_packed_device(data, offsets, sizes, w, h, c, d, max_file_size=max_file_size)
    status, out = status.cpu().numpy(), out.cpu().numpy()
    for i, f in enumerate(files):
        est, epx, *_ = oracle.decode(f, d) if expect is None else expect[i]
        assert status[i] == est, (w, h, c, d, i, status[i], est)
        if est == 0:
            assert np.array_equal(out[i].reshape(-1), epx), (w, h, c, d, i)
    return status


def test_decode_parity_packed(gpu, oracle):
    seen = set()
    for chans in (3, 4):
        for i, (w, h) in enumerate(SHAPES):
            files = [oracle.encode(imagegen.make(k, w, h, chans, 200 + i), w, h, chans, flags) for k in KINDS for flags in (0, 1, 2)]
            # container failures in the same call as the good files
            bad = bytearray(files[1]); bad[17] ^= 1                            # IHDR CRC
            files += [bytes(bad), files[2][:40], files[3][:-20], b"\0" + files[4][1:]]
            for d in (3, 4):
                seen.update(check_packed(gpu, oracle, files, w, h, chans, d).tolist())
    assert {0, 3, 4, 7} <= seen, seen
    rs = np.random.RandomState(7)
    for (kind, w, h, c, flags) in (("g1", 97, 13, 4, 0), ("g0", 200, 20, 3, 0), ("g1", 64, 16, 3, 1), ("g2", 31, 9, 4, 0)):
        png = oracle.encode(imagegen.make(kind, w, h, c, 2), w, h, c, flags)
        files = [png]
        for _ in range(120):
            bad = bytearray(png); bad[int(rs.randint(0, len(bad)))] ^= 1 << int(rs.randint(0, 8))
            files.append(bytes(bad))
        for d in (3, 4):
            st = check_packed(gpu, oracle, files, w, h, c, d)
            assert (st == 0).sum() > 1 and (st == 1).sum() > 0, (kind, np.unique(st))


def test_decode_reference_written_files_packed(gpu, oracle):
    """reference-written files (the oracle's encoder is byte-identical to the reference's: test_oracle_cpu / refreplay)"""
    for (kind, w, h, c) in (("g1", 640, 200, 3), ("g1", 640, 200, 4), ("g0", 1024, 128, 4), ("runs", 800, 60, 3), ("g2", 100, 40, 4)):
        img = imagegen.make(kind, w, h, c, 11)
        files = [oracle.encode(img, w, h, c, flags) for flags in (0, 1, 2)]
        for d in (3, 4):
            assert (check_packed(gpu, oracle, files, w, h, c, d) == 0).all()


@pytest.mark.parametrize("pre_roll", [256, 0])
def test_hand_built_streams_packed(gpu, L, oracle, pre_roll):
    """a sample of tests/streamgen.py's files, grouped by shape: packed decode == the oracle (but for the two documented
    deviations, NOT_FPNG), and the link pass repairs exactly as many subsequences as decode_batch_device on the same files"""
    import torch
    import streamgen
    assert L.fpngb_debug_decode_preroll(pre_roll) == 0
    groups = {}
    for name, f, chans, deflate_ok, deviation, data in streamgen.cases()[::3]:
        info = gpu.get_info_ex(f)
        key = info[1:4] if info[0] == 0 else None
        groups.setdefault(key, []).append((name, f, deviation))
    assert len(groups) > 1
    for key, items in groups.items():
        if key is None:
            continue
        w, h, c = key
        files = [f for _, f, _ in items]
        for d in (3, 4):
            expect = []
            for name, f, deviation in items:
                est, epx, *_ = oracle.decode(f, d)
                expect.append((gpu.FPNG_DECODE_NOT_FPNG, None) if deviation else (est, epx))
            L.fpngb_debug_decode_repairs(1)
            check_packed(gpu, oracle, files, w, h, c, d, expect=expect, max_file_size=max(len(f) for f in files))
            torch.cuda.synchronize()
            rep_packed = int(L.fpngb_debug_decode_repairs(1))
            t, stride, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, "cuda")
            gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d)
            torch.cuda.synchronize()
            assert int(L.fpngb_debug_decode_repairs(1)) == rep_packed, (key, d)


# ---- 3. equivalence with the strided call --------------------------------------------------------------------------------
def test_strided_offsets_equal_decode_batch_device(gpu, L, oracle):
    import torch
    rs = np.random.RandomState(5)
    for (w, h, c, n, flags) in ((640, 36, 3, 5, 0), (256, 40, 4, 7, 0), (130, 20, 4, 3, 1), (96, 8, 3, 3, 2), (1000, 120, 3, 4, 1)):
        files = [oracle.encode(imagegen.make(["g1", "g0", "runs", "g2", "mut"][i % 5], w, h, c, i), w, h, c, flags) for i in range(n)]
        for i in range(n):                                                   # stream damage behind an intact container
            st, _, _, _, io, il = gpu.get_info_ex(files[i])
            bad = bytearray(files[i]); pos = io + 8 + int(rs.randint(0, il)); bad[pos] ^= 1 << int(rs.randint(0, 8))
            files.append(bytes(bad))
        t, stride, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, "cuda")
        m = len(files)
        offsets = torch.arange(m, dtype=torch.int64, device="cuda") * stride
        dsizes = torch.from_numpy(sizes.view(np.int32).copy()).cuda()
        for d in (3, 4):
            a_px, a_st = gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d)
            b_px = torch.full((m, h, w, d), 0x5A, dtype=torch.uint8, device="cuda")
            _, b_st = gpu.decode_packed_device(t.reshape(-1), offsets, dsizes, w, h, c, d, out=b_px)
            torch.cuda.synchronize()
            a_st, b_st = a_st.cpu().numpy(), b_st.cpu().numpy()
            assert np.array_equal(a_st, b_st), (w, h, c, d, a_st, b_st)
            assert set(a_st.tolist()) <= {0, 1} and (a_st == 0).sum() >= n
            ok = torch.from_numpy(a_st == 0).cuda()
            assert torch.equal(a_px[ok], b_px[ok]), (w, h, c, d)


# ---- 4. shape and argument statuses in one call --------------------------------------------------------------------------
def test_shape_and_argument_statuses(gpu, oracle):
    import torch
    w, h, c = 64, 16, 4
    enc = lambda k, ww, hh, cc, s: oracle.encode(imagegen.make(k, ww, hh, cc, s), ww, hh, cc, 0)
    good = [enc("g1", w, h, c, s) for s in range(3)]
    other = [enc("g1", w + 1, h, c, 7), enc("g0", w, h + 1, c, 8), enc("g1", w, h, 3, 9)]
    max_size = max(len(f) for f in good + other)
    big = good[0][:33] + _chunk(b"tEXt", bytes(max_size)) + good[0][33:]    # valid, same shape, larger than max_file_size
    entries = [(good[0], 0), (other[0], SHAPE_MISMATCH), (good[1], 0), (other[1], SHAPE_MISMATCH),
               (other[2], SHAPE_MISMATCH), (b"", INVALID_ARG), (big, INVALID_ARG), (good[2], "misaligned"), (good[2], 0)]
    files = [f for f, _ in entries]
    buf, offs = pack(files)
    # the eighth file again, 2 bytes past a 4-byte boundary
    mis = len(buf) + 16 + 2
    buf = np.concatenate([buf, np.zeros(18, np.uint8), np.frombuffer(good[2], np.uint8)])
    offs[7] = mis
    sizes = [len(f) for f in files]
    data, offsets, dsizes = to_device(buf, offs, sizes)
    for d in (3, 4):
        out = torch.full((len(files), h, w, d), 0xA5, dtype=torch.uint8, device="cuda")
        _, status = gpu.decode_packed_device(data, offsets, dsizes, w, h, c, d, max_file_size=max_size, out=out)
        torch.cuda.synchronize()
        status, out = status.cpu().numpy(), out.cpu().numpy()
        for i, (f, want) in enumerate(entries):
            want = INVALID_ARG if want == "misaligned" else want
            assert status[i] == want, (d, i, status[i], want)
            if want == 0:
                assert np.array_equal(out[i].reshape(-1), oracle.decode(f, d)[1]), (d, i)
            else:
                assert (out[i] == 0xA5).all(), (d, i)                        # rows of failed files are left untouched


# ---- 5. emulated gather layout -------------------------------------------------------------------------------------------
def test_gather_layout(gpu, oracle):
    import torch
    w, h, c, nmax = 300, 40, 3, 5
    counts = [5, 3]                                                          # rank 1 leaves two slots unused
    files, slots = [], []
    for r, cnt in enumerate(counts):
        for i in range(nmax):
            f = oracle.encode(imagegen.make(["g1", "g0", "g2", "runs"][(r + i) % 4], w, h, c, 10 * r + i), w, h, c, i % 3) if i < cnt else b""
            slots.append(f)
    sizes = np.array([len(f) for f in slots], np.uint64)
    padded = (sizes + 15) // 16 * 16                                          # gather_offsets_kernel: exclusive scan of 16-byte aligned sizes
    offs = np.concatenate([[0], np.cumsum(padded)]).astype(np.int64)
    buf = np.zeros(int(offs[-1]), np.uint8)
    for o, f in zip(offs, slots):
        buf[o:o + len(f)] = np.frombuffer(f, np.uint8)
    data, offsets, dsizes = to_device(buf, offs, sizes)
    for d in (3, 4):
        out, status = gpu.decode_packed_device(data, offsets, dsizes, w, h, c, d)
        torch.cuda.synchronize()
        status, out = status.cpu().numpy(), out.cpu().numpy()
        for k, f in enumerate(slots):
            if not f:
                assert status[k] == INVALID_ARG, k
            else:
                assert status[k] == 0 and np.array_equal(out[k].reshape(-1), oracle.decode(f, d)[1]), (k, d)


# ---- 6. device-only round trip at full size ------------------------------------------------------------------------------
def test_device_round_trip_full_size(gpu):
    import torch
    from fpng_b200 import dist
    for (w, h, c, flags) in ((1920, 1080, 3, 0), (3840, 2160, 4, 0), (2048, 2048, 3, 1)):
        imgs = np.stack([imagegen.make(k, w, h, c, 4) for k in ("g1", "g0", "g2")])
        dev = torch.from_numpy(imgs).cuda()
        out, sizes = gpu.encode_batch_device(dev, flags)
        flat, offsets = dist.compact(out, sizes)
        px, status = gpu.decode_packed_device(flat, offsets, sizes, w, h, c, c)
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all()
        assert torch.equal(px, dev)
        info = gpu.get_info_batch_device(flat, offsets, sizes).cpu().numpy()
        assert (info[:, :4] == [0, w, h, c]).all()


# ---- 7. no host synchronisation ------------------------------------------------------------------------------------------
def test_no_host_synchronisation(gpu, oracle):
    import torch
    w, h, c = 512, 64, 4
    files = [oracle.encode(imagegen.make("g1", w, h, c, i), w, h, c, 0) for i in range(6)]
    data, offsets, sizes = packed_device(files)
    gpu.decode_packed_device(data, offsets, sizes, w, h, c, c)             # workspace reserved before the timed call
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)                                           # ~0.5 s of GPU time in front of the calls
        info = gpu.get_info_batch_device(data, offsets, sizes)
        px, status = gpu.decode_packed_device(data, offsets, sizes, w, h, c, c)
        assert not s.query(), "a call waited for the stream"
    s.synchronize()
    assert (status.cpu().numpy() == 0).all() and (info.cpu().numpy()[:, 0] == 0).all()
    for i, f in enumerate(files):
        assert np.array_equal(px[i].cpu().numpy().reshape(-1), oracle.decode(f, c)[1]), i
