"""CPU tests of the LZ77 oracle (tests/cpp/lz77_oracle.c): its files decode with zlib and PIL back to the input, and its parse
reaches each construct of the rule (include/fpng_b200.h "LZ77") that the GPU tests compare against."""
import io
import zlib

import numpy as np
import pytest

import lz77_oracle as lo


def idat(data: bytes) -> bytes:
    at, out = 8, b""
    while at < len(data):
        n = int.from_bytes(data[at:at + 4], "big")
        if data[at + 4:at + 8] == b"IDAT":
            out += data[at + 8:at + 8 + n]
        at += 12 + n
    return out


@pytest.mark.parametrize("c", [1, 2, 3, 4])
@pytest.mark.parametrize("K", [1, 8, 128])
def test_files_decode_with_pil(c, K):
    from PIL import Image
    rs = np.random.default_rng(c * 10 + K)
    img = np.tile(rs.integers(0, 256, (5, 7, c), dtype=np.uint8), (20, 30, 1))
    img[30:32] = rs.integers(0, 256, (2, img.shape[1], c))
    data = lo.png_encode(img, K)
    assert np.array_equal(np.array(Image.open(io.BytesIO(data))).reshape(img.shape), img)
    assert len(zlib.decompress(idat(data))) == (img.shape[1] * c + 1) * img.shape[0]


@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_16bit_stream_decodes(c):
    rs = np.random.default_rng(c)
    img = np.tile(rs.integers(0, 65536, (3, 5, c), dtype=np.uint16), (10, 10, 1))
    data = lo.png_encode(img, 8)
    assert len(zlib.decompress(idat(data))) == (img.shape[1] * 2 * c + 1) * img.shape[0]


@pytest.mark.parametrize("depth,K", [(1, 0), (2, 0), (4, 0), (8, 0), (8, 3), (2, 4), (8, 200)])
def test_labels_decode(depth, K):
    """palette files give their indices back through PIL; gray files inflate to the packed rows"""
    from PIL import Image
    rs = np.random.default_rng(depth)
    pal = None if K == 0 else rs.integers(0, 256, (K, 3), dtype=np.uint8)
    ids = np.tile(rs.integers(0, (1 << depth) if K == 0 else K, (6, 9)), (11, 13))
    data = lo.label_encode(ids, depth, 8, pal)
    if pal is not None or depth == 8:
        assert np.array_equal(np.array(Image.open(io.BytesIO(data))).astype(np.int64), ids)
    rows, _ = lo.label_rows(ids, depth)
    assert len(zlib.decompress(idat(data))) == rows.size + rows.shape[0]


def info(rows, K=8, flags=0):
    return lo.encode_rows(rows.astype(np.uint8), 1, lo.container(rows.shape[1], rows.shape[0], 8, 0), K, flags, want_info=True)


def test_constructs_reached():
    rs = np.random.default_rng(0)
    rand = rs.integers(0, 2, (4, 40)) * 128
    _, d = info(np.concatenate([rand, rand, rand]))
    assert d["rows_crossed"] > 0
    _, d = info(np.zeros((4, 600)))                                    # long runs: 258-byte matches across rows
    assert d["len258"] > 0 and d["rows_crossed"] > 0
    _, d = info(np.tile(np.random.default_rng(0).integers(0, 2, (1, 300)) * 128, (1, 200)))
    assert d["cut_at_segment"] > 0
    for n in (16383, 16384, 16385, 3 * 16384 + 1):
        data, d = info(np.tile(rs.integers(0, 2, (1, 300)) * 128, (1, n // 300 + 1))[:, :n - 1])
        assert d["n"] == n and len(zlib.decompress(idat(data))) == n


def test_distance_symbols_zero_and_one():
    _, d = info(np.random.default_rng(5).integers(0, 256, (1, 40)))
    assert d["dist_syms"] == 0
    data, d = info(np.full((1, 100), 128))
    assert d["dist_syms"] == 1
    assert zlib.decompress(idat(data)) == bytes([1, 128]) + bytes(99)     # the Sub filter wins


def test_stored_fallback():
    rs = np.random.default_rng(1)
    data, d = info(rs.integers(0, 256, (64, 64)))
    assert d["stored"] == 1 and d["zcomp"] > d["zstored"]
    data, d = info(np.zeros((8, 8)), flags=2)
    assert d["stored"] == 1
    assert zlib.decompress(idat(data)) == bytes(72)


def at(toks, pos):
    """the token that starts at stream position pos"""
    p = 0
    for t in toks:
        if p == pos:
            return t
        p += t[0] if isinstance(t, tuple) else 1
    raise AssertionError(pos)


def test_window_edge():
    """a source exactly 32768 bytes back is taken; one 32769 bytes back is not (the rule's p - q > 32768)"""
    rs = np.random.default_rng(7)
    x = rs.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    assert at(lo.parse(x + x[:100], 8), 32768) == (100, 32768)
    toks = lo.parse(x + b"\x00" + x[:100], 8)
    assert at(toks, 32769) == x[0] and all(t[1] <= 32768 for t in toks if isinstance(t, tuple))


def colliding_triples():
    """two different 3-byte strings of one hash, found from the formula H(p) = (v * 0x9E3779B1 mod 2^32) >> 17"""
    seen = {}
    for v in range(1 << 24):
        h = ((v * 0x9E3779B1) & 0xFFFFFFFF) >> 17
        if h in seen:
            return seen[h].to_bytes(3, "big"), v.to_bytes(3, "big")
        seen[h] = v
    raise AssertionError


COLLIDING = colliding_triples()


def collision_stream():
    """a, filler, b, filler, a with H(a) = H(b): the last a's nearest chain entry is the collision b, the next one the real a"""
    a, b = COLLIDING
    return a + bytes([11, 13, 17, 19]) + b + bytes([23, 29, 31]) + a


def test_collision_counts_toward_k():
    s = collision_stream()
    p = len(s) - 3
    k1, k2 = lo.parse(s, 1), lo.parse(s, 2)
    assert k1[-3:] == list(s[p:])                                     # K = 1 walks only the collision: literals
    assert k2[-1] == (3, p)                                           # K = 2 reaches the real a at distance p


def test_ties_go_to_the_nearest():
    rs = np.random.default_rng(8)
    a = rs.integers(0, 256, 8, dtype=np.uint8).tobytes()
    s = a + b"\x01\x02" + a + b"\x03\x04" + a
    assert lo.parse(s, 8)[-1] == (8, 10)


TIE = (0, 48, 1500)                                                   # seed, leading zero bytes, row length: zcomp == zstored


def tie_row():
    seed, k, R = TIE
    row = np.random.default_rng(seed).integers(0, 256, (1, R), dtype=np.uint8)
    row[0, :k] = 0
    return row


def test_compressed_equals_stored_keeps_compressed():
    row = tie_row()
    data, d = lo.encode_rows(row, 1, lo.container(row.shape[1], 1, 8, 0), 8, 0, want_info=True)
    assert d["zcomp"] == d["zstored"] and d["stored"] == 0
    assert zlib.decompress(idat(data))[1:] == row.tobytes() or len(zlib.decompress(idat(data))) == row.size + 1


def test_api_rejects_bad_depth():
    import fpng_b200
    with pytest.raises(ValueError):
        fpng_b200.encode_png_device([], lz77=300)
    with pytest.raises(ValueError):
        fpng_b200.encode_labels_device([], lz77=-1)


# The size table (tests/lz77_sizes.py), first two images of each workload, total bytes.  The lz77_* and run_only columns are the
# exact oracles' and hold everywhere; the PIL and cv2 columns hold for the library versions in SIZE_LIBS.
SIZE_LIBS = ("12.2.0", "4.13.0", "1.3")
SIZES = {
    "E1": {"lz77_8": 24703, "lz77_32": 24819, "lz77_128": 24800, "run_only": 21242, "pil_6": 24976, "pil_1": 37406, "cv2_6": 24991, "cv2_1": 37479},
    "E2": {"lz77_8": 411171, "lz77_32": 394793, "lz77_128": 388112, "run_only": 432351, "pil_6": 391872, "pil_1": 426708, "cv2_6": 396802, "cv2_1": 426875},
    "E3": {"lz77_8": 608928, "lz77_32": 598099, "lz77_128": 597055, "run_only": 481148, "pil_6": 496181, "pil_1": 641670, "cv2_6": 570044, "cv2_1": 615905},
    "E4": {"lz77_8": 18571225, "lz77_32": 18324202, "lz77_128": 18137654, "run_only": 16313559, "pil_6": None, "pil_1": None, "cv2_6": 17887739, "cv2_1": 18970923},
    "V1": {"lz77_8": 10797, "lz77_32": 10858, "lz77_128": 10868, "run_only": 10584, "pil_6": 9022, "pil_1": 12224, "cv2_6": 9260, "cv2_1": 11962},
    "V2": {"lz77_8": 23457, "lz77_32": 23604, "lz77_128": 23541, "run_only": 20540, "pil_6": 24990, "pil_1": 31796, "cv2_6": 24991, "cv2_1": 37479},
    "V3": {"lz77_8": 12534, "lz77_32": 12409, "lz77_128": 12128, "run_only": 11109, "pil_6": 11835, "pil_1": 16187, "cv2_6": 16262, "cv2_1": 28537},
    "C2": {"lz77_8": 6638740, "lz77_32": 6448812, "lz77_128": 6421560, "run_only": 6803835, "pil_6": 5624803, "pil_1": 6658570, "cv2_6": 6308314, "cv2_1": 6670232},
}


def test_size_table():
    import cv2
    import PIL
    import lz77_sizes
    got = lz77_sizes.table(tuple(SIZES), 2)
    same_libs = (PIL.__version__, cv2.__version__, zlib.ZLIB_RUNTIME_VERSION) == SIZE_LIBS
    for name, want in SIZES.items():
        for arm, v in want.items():
            if arm.startswith(("lz77", "run_only")) or same_libs:
                assert got[name][arm] == v, (name, arm, got[name][arm], v)
