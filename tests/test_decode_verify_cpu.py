"""CPU tests of the decoder's opt-in integrity check (fpngb_set_decode_verify): the Adler-32 decomposition the verify kernel
(decode_adler_kernel) relies on, restated in numpy and compared with zlib, and the switch itself without a device."""
import zlib

import numpy as np
import pytest

M = 65521


def stream_of(delta, stored):
    """the inflated stream of an fpng file: per row the filter byte (0, then 2 in compressed files; 0 in stored files), then
    the row's delta bytes"""
    h, bpl = delta.shape
    filt = np.zeros((h, 1), np.uint8)
    if not stored:
        filt[1:] = 2
    return np.concatenate([filt, delta], axis=1).reshape(-1)


def adler_by_parts(delta, stored, row_cuts, col_cuts, row0=0, total_rows=None):
    """Adler-32 of stream_of(delta) from per-part sums: every (row range, column range) block adds sum x and sum i*x with its
    own positions, the filter bytes in closed form.  row0 / total_rows place the delta rows inside a taller stream whose other
    rows are all zero (positions past 2^32 without a 4 GiB array)."""
    h, bpl = delta.shape
    total_rows = h if total_rows is None else total_rows
    s1 = s2 = 0
    rb = [0] + sorted(row_cuts) + [h]
    cb = [0] + sorted(col_cuts) + [bpl]
    for r0, r1 in zip(rb, rb[1:]):
        for c0, c1 in zip(cb, cb[1:]):
            blk = delta[r0:r1, c0:c1].astype(np.int64)
            if blk.size == 0:
                continue
            rows = np.arange(r0 + row0, r1 + row0, dtype=object)[:, None]
            cols = np.arange(c0, c1, dtype=object)[None, :]
            pos = rows * (bpl + 1) + 1 + cols               # Python integers: no wrap past 2^63
            s1 = (s1 + int(blk.sum())) % M
            s2 = (s2 + int((pos * blk.astype(object)).sum())) % M
    if not stored and total_rows > 1:
        s1 = (s1 + 2 * (total_rows - 1)) % M
        s2 = (s2 + (bpl + 1) * total_rows * (total_rows - 1)) % M
    n = total_rows * (bpl + 1)
    a = (1 + s1) % M
    b = (n + n * s1 - s2) % M
    return (b << 16) | a


@pytest.mark.parametrize("seed", range(12))
def test_decomposition_equals_zlib(seed):
    rs = np.random.RandomState(seed)
    h, w, c = int(rs.randint(1, 40)), int(rs.randint(1, 70)), int(rs.choice([3, 4]))
    bpl = w * c
    delta = rs.randint(0, 256, size=(h, bpl)).astype(np.uint8)
    if seed % 3 == 0:
        delta[:] = 255                                       # the largest sums
    for stored in (False, True):
        want = zlib.adler32(stream_of(delta, stored).tobytes())
        rcuts = sorted(set(rs.randint(0, h + 1, size=rs.randint(0, 4)).tolist()))
        ccuts = sorted(set(rs.randint(0, bpl + 1, size=rs.randint(0, 4)).tolist()))
        assert adler_by_parts(delta, stored, rcuts, ccuts) == want
        assert adler_by_parts(delta, stored, list(range(1, h)), list(range(16, bpl, 16))) == want   # one warp per row, 16-byte vectors


def test_positions_past_2_32():
    """a stream longer than 2^32 bytes (a 2^24 x 64 RGBA file has 2^32 + 64 of them): the closed form with Python integers against
    zlib over the same stream built in pieces -- all-zero rows except a few rows at the end, so zlib can run over it by combining"""
    bpl = (1 << 24) * 4 // 1024                              # 64 Ki bytes per row; 2^16 + 4 rows pass 2^32 bytes
    total_rows = (1 << 16) + 4
    rs = np.random.RandomState(7)
    tail = rs.randint(0, 256, size=(3, bpl)).astype(np.uint8)
    row0 = total_rows - 3
    for stored in (False, True):
        # zlib over the whole stream, fed in rows (adler32 keeps its running state)
        a = 1
        zero_row = np.zeros(bpl, np.uint8).tobytes()
        for y in range(total_rows):
            f = b"\x00" if (stored or y == 0) else b"\x02"
            a = zlib.adler32(f + (tail[y - row0].tobytes() if y >= row0 else zero_row), a)
        assert total_rows * (bpl + 1) > 1 << 32
        assert adler_by_parts(tail, stored, [1, 2], [bpl // 3], row0=row0, total_rows=total_rows) == a


def test_switch_round_trip_without_device():
    import fpng_b200
    from fpng_b200._lib import lib
    try:
        assert fpng_b200.decode_verify() is False            # off at load
        fpng_b200.set_decode_verify(True)
        assert fpng_b200.decode_verify() is True
        assert lib().fpngb_get_decode_verify() == 1
        fpng_b200.set_decode_verify(False)
        assert fpng_b200.decode_verify() is False
        assert fpng_b200.FPNGB_DECODE_ADLER_MISMATCH == 102
    finally:
        fpng_b200.set_decode_verify(False)


def test_decode_entry_points_still_refuse_without_device():
    import ctypes as C

    import fpng_b200
    from fpng_b200._lib import lib
    if lib().fpngb_is_initialized():
        pytest.skip("the library was initialised on a device by an earlier test")
    png = bytes(range(64))
    fpng_b200.set_decode_verify(True)
    try:
        L = lib()
        out = np.zeros(16, np.uint8)
        st = L.fpngb_decode_host(png, len(png), out.ctypes.data_as(C.c_void_p), out.size, None, None, None, 3)
        assert st != 0
        rc = L.fpngb_decode_packed_device(1024, 1024, 1024, 1, 64, 4, 4, 3, 3, 1024, 48, 1024, None)
        assert rc == 3                                       # FPNGB_ERR_NOT_INITIALIZED
        rc = L.fpngb_decode_packed_ragged_device(1024, 64, 1024, 1024, 1, 64, 4, 4, 3, 1024, 48, 1024, None, 1024, None)
        assert rc == 3
    finally:
        fpng_b200.set_decode_verify(False)
