"""Hand-built fpng streams (tests/streamgen.py): tables and token sequences no encoder writes but the format allows (or that
break it in one specific way).  The oracle's status and pixels must equal the reference decoder's on every file, and
zlib.decompress must return the intended filtered stream for every file that is valid Deflate (an independent check that the
writer writes what the case says)."""
import struct
import zlib

import numpy as np
import pytest

import streamgen

CASES = streamgen.cases()


def idat(f: bytes) -> bytes:
    at = f.index(b"IDAT")
    return f[at + 4:at + 4 + struct.unpack(">I", f[at - 4:at])[0]]


def test_writer_agrees_with_zlib():
    assert len(CASES) > 150
    for name, f, chans, deflate_ok, deviation, data in CASES:
        if deflate_ok:
            assert zlib.decompress(idat(f)) == data, name
        else:
            with pytest.raises(zlib.error):
                zlib.decompress(idat(f))


def test_oracle_decodes_like_the_reference(oracle, ref):
    accepted = rejected = 0
    for name, f, chans, deflate_ok, deviation, data in CASES:
        for d in (3, 4):
            est, epx, *_ = oracle.decode(f, d)
            rst, rpx, *_ = ref.decode(f, d)
            assert est == rst, (name, d, est, rst)
            if est == 0:
                assert np.array_equal(epx, rpx), (name, d)
        accepted += est == 0
        rejected += est != 0
        if deviation:
            assert est == 0, name                                          # the reference accepts them
    assert accepted > 60 and rejected > 60
