"""GPU tests of the decoder's speculation repair (decode_scan_kernel's guessed subsequence starts, decode_link_kernel's chain
check and re-decode, the carry between its 1024-subsequence chunks).  Pixels and statuses must equal the oracle's, and the
device's repair count (fpngb_debug_decode_repairs) must equal the CPU model's (test_decoder_model_cpu.Model.link_parallel) for
the same file and pre-roll: a different count with the same pixels means one of the two restatements of the link loop is wrong.

Slow-synchronising files (imagegen "u<k>", 2-pass) make most subsequence guesses wrong at the default pre-roll; pre-roll 0, 1
and 13 (fpngb_debug_decode_preroll) force wrong guesses on the ordinary decode corpus."""
import numpy as np
import pytest

import imagegen
from common import with_text_chunk
from test_decoder_model_cpu import K_PRE_ROLL, Model, model_repairs

pytestmark = pytest.mark.gpu


@pytest.fixture
def L(gpu):
    from fpng_b200._lib import lib
    L = lib()
    yield L
    L.fpngb_debug_decode_preroll(K_PRE_ROLL)                                 # the default


def decode_counted(gpu, L, png, desired):
    """(status, pixels, link repairs of this one decode)"""
    L.fpngb_debug_decode_repairs(1)
    st, px, *_ = gpu.fpng_decode_memory(png, desired)
    return st, px, int(L.fpngb_debug_decode_repairs(1))


def check_file(gpu, L, oracle, png, pre_roll=K_PRE_ROLL, desired=(3, 4), want=None):
    """decodes `png` at every desired channel count: statuses / pixels against the oracle, repairs against the model (`want`:
    already known); returns the repair count"""
    if want is None:
        want = model_repairs(png, pre_roll)
    for d in desired:
        est, epx, *_ = oracle.decode(png, d)
        st, px, rep = decode_counted(gpu, L, png, d)
        assert st == est, (len(png), pre_roll, d, st, est)
        if st == 0:
            assert np.array_equal(px, epx), (len(png), pre_roll, d)
        assert rep == want, (len(png), pre_roll, d, rep, want)
    return want


SLOW = [("u128", 1024, 160, 3, 1), ("u128", 1920, 200, 3, 1), ("u128", 1024, 160, 4, 1), ("u64", 1024, 160, 4, 1),
        ("u16", 1024, 160, 4, 1), ("u16", 1920, 200, 3, 0), ("u2", 1024, 160, 4, 0)]


@pytest.mark.parametrize("kind,w,h,chans,flags", SLOW)
def test_slow_synchronising_files(gpu, L, oracle, kind, w, h, chans, flags):
    img = imagegen.make(kind, w, h, chans, 1)
    png = oracle.encode(img, w, h, chans, flags)
    assert png[60] & 6, "dynamic block"                                    # not the stored-block fallback
    rs = np.random.RandomState(w + h + chans)
    for pad in range(4):                                                   # all four alignments of the zlib stream inside its word
        f = png if pad == 0 else with_text_chunk(png, pad)
        m = Model(f, gpu.get_info_ex(f))
        ok, _, repairs, iters = m.link_parallel(m.scan_all())
        assert ok and len(iters) >= 2                                       # several 1024-subsequence chunks
        if flags == 1 and kind in ("u128", "u64"):
            assert repairs > (m.g1 - m.g0) // 2 and max(iters) >= 3, (repairs, iters)
        check_file(gpu, L, oracle, f, want=repairs)
        np.testing.assert_array_equal(gpu.fpng_decode_memory(f, chans)[1], img.reshape(-1))
        # a corrupted copy: a bit flip after the header
        bad = bytearray(f); pos = int(rs.randint(60 + (12 + pad if pad else 0), len(bad))); bad[pos] ^= 1 << int(rs.randint(0, 8))
        check_file(gpu, L, oracle, bytes(bad))


def test_batch_mixes_slow_and_ordinary_files(gpu, L, oracle):
    import torch
    for (w, h, c, flags) in ((1024, 160, 3, 1), (1024, 160, 4, 1)):
        kinds = ["u128", "g1", "u64", "g1", "u16", "u2"]
        files = [oracle.encode(imagegen.make(k, w, h, c, i), w, h, c, flags) for i, k in enumerate(kinds)]
        files[3] = bytes(files[3][:200]) + bytes([files[3][200] ^ 4]) + files[3][201:]     # a corrupted one among them
        want = sum(model_repairs(f) for f in files)
        t, stride, sizes, ofs, lens, ww, hh, cc = gpu.pack_files_for_device(files, "cuda")
        for d in (3, 4):
            L.fpngb_debug_decode_repairs(1)
            out, status = gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d)
            torch.cuda.synchronize()
            assert int(L.fpngb_debug_decode_repairs(1)) == want
            status, out = status.cpu().numpy(), out.cpu().numpy()
            for i in range(len(files)):
                est, epx, *_ = oracle.decode(files[i], d)
                assert status[i] == est, (i, status[i], est)
                if est == 0:
                    assert np.array_equal(out[i].reshape(-1), epx), (w, h, c, i, d)
        assert want > 0


def test_ordinary_file_needs_no_repair(gpu, L, oracle):
    """at the default pre-roll the prefix code locks on almost always: no repairs on these 1024x160 g1 files and a handful on
    the larger ones, on the device as in the model"""
    for (w, h, c, flags, most) in ((1024, 160, 3, 0, 0), (1024, 160, 4, 0, 0), (1920, 200, 3, 0, 8), (1920, 200, 3, 1, 8)):
        png = oracle.encode(imagegen.make("g1", w, h, c, 1), w, h, c, flags)
        repairs = check_file(gpu, L, oracle, png)
        assert repairs <= most, (w, h, c, flags, repairs)


# ---- forced wrong guesses on the ordinary decode corpus (test_decode_gpu.py's shapes, corrupted streams and write-path cases)
SHAPES = [(1, 1), (2, 2), (5, 3), (63, 3), (85, 2), (129, 6), (257, 33), (512, 64), (687, 41), (2049, 2)]


@pytest.mark.parametrize("pre_roll", [0, 1, 13])
def test_forced_wrong_guesses(gpu, L, oracle, pre_roll):
    assert L.fpngb_debug_decode_preroll(K_PRE_ROLL + 1) != 0               # beyond the scan kernel's window: refused
    assert L.fpngb_debug_decode_preroll(pre_roll) == 0
    total = 0
    for kind in ("g1", "runs"):
        for chans in (3, 4):
            for i, (w, h) in enumerate(SHAPES):
                img = imagegen.make(kind, w, h, chans, 200 + i)
                for flags in (0, 1, 2):
                    total += check_file(gpu, L, oracle, oracle.encode(img, w, h, chans, flags), pre_roll)
    rs = np.random.RandomState(7)
    for (kind, w, h, c, flags) in (("g1", 97, 13, 4, 0), ("g0", 200, 20, 3, 0), ("g1", 64, 16, 3, 1)):
        png = oracle.encode(imagegen.make(kind, w, h, c, 2), w, h, c, flags)
        for t in range(40):
            bad = bytearray(png); bad[int(rs.randint(0, len(bad)))] ^= 1 << int(rs.randint(0, 8))
            check_file(gpu, L, oracle, bytes(bad), pre_roll, desired=(c,))
    for (kind, w, h, c, flags) in (("g1", 700, 200, 3, 0), ("mut", 1000, 120, 3, 1), ("runs", 640, 200, 4, 0), ("g1", 3, 3000, 4, 0)):
        png = oracle.encode(imagegen.make(kind, w, h, c, 5), w, h, c, flags)
        total += check_file(gpu, L, oracle, png, pre_roll)
        bad = bytearray(png); pos = int(rs.randint(60, len(bad))); bad[pos] ^= 1 << int(rs.randint(0, 8))
        check_file(gpu, L, oracle, bytes(bad), pre_roll)
    assert total > 1000                                                    # the guesses really were wrong


@pytest.mark.parametrize("pre_roll", [K_PRE_ROLL, 0])
def test_hand_built_streams(gpu, L, oracle, pre_roll):
    """tests/streamgen.py's files (other tables, HLIT / HDIST / HCLEN values, every length symbol, broken token sequences):
    status and pixels as the oracle's (== the reference's, tests/test_streamgen_cpu.py), except the two documented deviations
    (INTEGRATION.md section 7), which the GPU rejects where the reference decodes them"""
    import streamgen
    assert L.fpngb_debug_decode_preroll(pre_roll) == 0
    for name, f, chans, deflate_ok, deviation, data in streamgen.cases():
        want = model_repairs(f, pre_roll)
        for d in (3, 4):
            est, epx, *_ = oracle.decode(f, d)
            st, px, rep = decode_counted(gpu, L, f, d)
            if deviation:
                assert est == 0 and st == gpu.FPNG_DECODE_NOT_FPNG, (name, d, st)
            else:
                assert st == est, (name, pre_roll, d, st, est)
                if st == 0:
                    assert np.array_equal(px, epx), (name, pre_roll, d)
            assert rep == want, (name, pre_roll, d, rep, want)
