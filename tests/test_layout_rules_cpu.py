"""The argument rules every device entry point shares (fpng_b200/csrc/layout.h), compiled with g++ into a small driver
(tests/cpp/layout_test.cpp) and checked against a restatement, in Python, of the rule sets of the calls that use them:
  * u8:  a uint8 input (the strided and ragged encodes): interleaved or planar, inside the address space, 32-bit row pitch;
  * in:  a float input (the typed encodes): the same in elements, the base and strides aligned to the element size, and every
         stride inside 64 bits once scaled back to bytes;
  * out: an output (the decodes): as a float input, and no two elements share a byte.  The image stride of an output batch of one
         addresses nothing and is not checked when scaled back to bytes (it may wrap), as the decodes have always done.
The format parser is checked the same way."""
import os
import random
import struct
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = (1 << 64) - 1
OK, INVALID, ALIGNMENT = 0, 1, 5


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("layout") / "layout_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "layout_test.cpp"), "-o", exe])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return [tuple(line.split()) for line in out.splitlines()]
    return run


def classify(image, row, pixel, chan, n, h, w, c):
    """classify_layout with the C++ uint64 arithmetic: canonical strides of size-1 dimensions, or None"""
    if w == 1:
        pixel = c if chan == 1 else 1
    inter = pixel == c and chan == 1
    planar = not inter and pixel == 1 and chan >= 1
    if not (inter or planar):
        return None
    if h == 1:
        row = w * c if inter else w
    if n == 1:
        image = (h * row) & M
    return [image, row, pixel, chan, planar]


def span(base, L, n, h, w, c):
    """offset of the last element's first byte, or None when it wraps the address space"""
    s = sum((k - 1) * v for k, v in zip((n, h, w, c), L[:4]))
    return None if s > M - base else s


def disjoint(L, n, h, w, c):
    dims = sorted((v, k) for k, v in zip((n, h, w, c), L[:4]) if k > 1)
    extent = 0
    for st, k in dims:
        if st < extent + 1:
            return False
        extent += st * (k - 1)
    return True


def rule_u8(base, image, row, pixel, chan, n, h, w, c, elem):
    """the uint8 encodes: classify, a 32-bit row pitch, the span"""
    L = classify(image, row, pixel, chan, n, h, w, c)
    if L is None or L[1] > 0xFFFFFFFF or span(base, L, n, h, w, c) is None:
        return INVALID, None
    return OK, L


def rule_in(base, image, row, pixel, chan, n, h, w, c, es):
    """the typed encodes: alignment, classify in elements, no stride past 64 bits in bytes, the span"""
    if any(v % es for v in (base, image, row, pixel, chan)):
        return ALIGNMENT, None
    E = classify(image // es, row // es, pixel // es, chan // es, n, h, w, c)
    if E is None or any(v > M // es for v in E[:4]):
        return INVALID, None
    L = [v * es for v in E[:4]] + [E[4]]
    last = span(base, L, n, h, w, c)
    if last is None or last > M - base - (es - 1):
        return INVALID, None
    return OK, L


def rule_out(base, image, row, pixel, chan, n, h, w, c, es):
    """the decodes: alignment, classify and disjointness in elements, strides scaled back with uint64 wrap, the span"""
    if any(v % es for v in (base, image, row, pixel, chan)):
        return ALIGNMENT, None
    E = classify(image // es, row // es, pixel // es, chan // es, n, h, w, c)
    if E is None or not disjoint(E, n, h, w, c):
        return INVALID, None
    L = [(v * es) & M for v in E[:4]] + [E[4]]
    last = span(base, L, n, h, w, c)
    if last is None or last > M - base - (es - 1):
        return INVALID, None
    return OK, L


RULES = {"u8": rule_u8, "in": rule_in, "out": rule_out}


def check_layouts(driver, cases):
    got = driver(["L " + " ".join(str(v) for v in case) for case in cases])
    assert len(got) == len(cases)
    verdicts = set()
    for case, g in zip(cases, got):
        mode, args = case[0], case[1:]
        rc, L = RULES[mode](*args)
        want = (str(rc),) if rc else (str(rc),) + tuple(str(v) for v in L[:4]) + (str(int(L[4])),)
        assert g[:len(want)] == want, (case, want, g)
        verdicts.add((mode, rc))
    return verdicts


def strides_for(rng, n, h, w, c, es):
    """byte strides of a layout that is tight, pitched, planar, broadcast, misaligned, huge or just random"""
    kind = rng.randrange(8)
    if kind == 0:                                                   # tight interleaved
        return h * w * c * es, w * c * es, c * es, es
    if kind == 1:                                                   # pitched interleaved, images apart or broadcast
        row = (w * c + rng.randrange(0, 40)) * es
        return rng.choice([h * row, 0, h * row + es * rng.randrange(1, 9)]), row, c * es, es
    if kind == 2:                                                   # planar CHW or HCW
        if rng.randrange(2):
            return c * h * w * es, w * es, es, h * w * es
        return h * c * w * es, c * w * es, es, w * es
    if kind == 3:                                                   # overlapping rows or planes
        return rng.choice([0, w * es]), rng.choice([0, es, w * es]), rng.choice([es, c * es]), rng.choice([es, w * es, 0])
    if kind == 4:                                                   # misaligned by one to es - 1 bytes somewhere
        s = [h * w * c * es, w * c * es, c * es, es]
        s[rng.randrange(4)] += rng.randrange(1, max(es, 2))
        return tuple(s)
    if kind == 5:                                                   # strides near the top of 64 bits
        big = M - rng.randrange(0, 1 << 20)
        return rng.choice([big, h * w * c * es]), rng.choice([big // h if h else big, w * c * es, 1 << 63]), c * es, es
    if kind == 6:                                                   # small random values
        return tuple(rng.randrange(0, 64) for _ in range(4))
    return tuple(rng.choice([0, 1, 2, 3, 4, 8, 12, 16, es * c, es * w, es * w * c, 1 << 32, 1 << 62, M]) for _ in range(4))


def random_cases(seed, count):
    rng = random.Random(seed)
    cases = []
    for _ in range(count):
        mode = rng.choice(["u8", "in", "out"])
        es = 1 if mode == "u8" else rng.choice([1, 2, 4]) if mode == "out" else rng.choice([2, 4])
        n, h, w = (rng.choice([1, 1, 2, 3, 7, 65535]) for _ in range(3))
        c = rng.choice([3, 4])
        base = rng.choice([0x7F0000000000, 0x7F0000000000 + rng.randrange(1, 16), M - rng.randrange(0, 1 << 40), rng.randrange(0, 1 << 48)])
        cases.append((mode, base) + tuple(strides_for(rng, n, h, w, c, es)) + (n, h, w, c, es))
    return cases


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_layouts_match_each_calls_rules(driver, seed):
    verdicts = check_layouts(driver, random_cases(seed, 4000))
    for mode in ("u8", "in", "out"):
        assert (mode, OK) in verdicts and (mode, INVALID) in verdicts        # every rule set both accepts and rejects
    assert ("in", ALIGNMENT) in verdicts and ("out", ALIGNMENT) in verdicts


def test_edge_cases(driver):
    base = 0x7F0000000000
    cases = []
    for mode, sizes in (("u8", [1]), ("in", [2, 4]), ("out", [1, 2, 4])):
        for es in sizes:
            for c in (3, 4):
                n, h, w = 2, 3, 5
                tight = (h * w * c * es, w * c * es, c * es, es)
                planar = (c * h * w * es, w * es, es, h * w * es)
                for dims in ((1, h, w), (n, 1, w), (n, h, 1), (1, 1, 1), (1, 1, w), (n, 1, 1)):     # size-1 dimensions everywhere
                    for s in (tight, planar, (12345 * es, 7 * es, 3 * es, 11 * es), (0, 0, 0, 0)):
                        cases.append((mode, base) + s + dims + (c, es))
                for k in range(4):                                                              # stride 0 in each position
                    for s in (tight, planar):
                        z = list(s)
                        z[k] = 0
                        cases.append((mode, base) + tuple(z) + (n, h, w, c, es))
                for off in range(1, 4):                                                         # misaligned base or stride
                    cases.append((mode, base + off) + tight + (n, h, w, c, es))
                    for k in range(4):
                        z = list(tight)
                        z[k] += off
                        cases.append((mode, base) + tuple(z) + (n, h, w, c, es))
                top = M - (h * w * c * es) * n                                                  # spans that end at or wrap past 2^64
                for b in (top - es, top - es + 1, top, top + 1, top + es, M - es + 1):
                    b -= b % es
                    cases.append((mode, b) + tight + (n, h, w, c, es))
                cases.append((mode, base) + (1 << 63, 1 << 62, c * es, es) + (n, h, w, c, es))  # 64-bit strides
                cases.append((mode, base) + (M - M % es, w * c * es, c * es, es) + (n, h, w, c, es))
    check_layouts(driver, cases)


def test_batch_of_one_whose_canonical_image_stride_passes_64_bits(driver):
    """n == 1, h == 2 and a 2^63-byte row pitch: the canonical image stride h * row does not fit in 64 bits.  A float input is
    refused (its strides must fit once scaled back to bytes); an output accepts it (the image stride of one image addresses
    nothing); a uint8 input is refused for its row pitch."""
    base = 0x1000
    row = 1 << 63
    for mode, es in (("in", 4), ("in", 2), ("out", 4), ("out", 2), ("out", 1), ("u8", 1)):
        check_layouts(driver, [(mode, base, 0, row, 3 * es, es, 1, 2, 4, 3, es)])
    assert rule_in(base, 0, row, 12, 4, 1, 2, 4, 3, 4)[0] == INVALID
    assert rule_out(base, 0, row, 12, 4, 1, 2, 4, 3, 4)[0] == OK
    assert rule_u8(base, 0, row, 3, 1, 1, 2, 4, 3, 1)[0] == INVALID


def fbits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def parse_rule(null, dtype, chans, scale, bias):
    """the typed calls' format rules: a float32 / float16 / bfloat16 dtype and finite scale and bias in the channels in use"""
    if null or dtype not in (1, 2, 3):
        return (INVALID,)
    used = min(chans, 4)
    if any(x in (0x7F800000, 0xFF800000) or (x & 0x7F800000) == 0x7F800000 for x in scale[:used] + bias[:used]):
        return (INVALID,)
    return (OK, dtype, 4 if dtype == 1 else 2) + tuple(scale[:used]) + (0,) * (4 - used) + tuple(bias[:used]) + (0,) * (4 - used)


def test_format_parser(driver):
    rng = random.Random(7)
    special = [fbits(v) for v in (0.0, -0.0, 1.0, -1.5, 127.5, 3.4e38, 1e-45)] + [0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001]
    cases = []
    for _ in range(3000):
        null = int(rng.random() < 0.05)
        dtype = rng.choice([0, 1, 2, 3, 4, 0xFFFFFFFF])
        chans = rng.choice([0, 1, 3, 4, 5])
        scale = [rng.choice(special) if rng.random() < 0.15 else fbits(rng.uniform(-300, 300)) for _ in range(4)]
        bias = [rng.choice(special) if rng.random() < 0.15 else fbits(rng.uniform(-300, 300)) for _ in range(4)]
        cases.append((null, dtype, chans, scale, bias))
    got = driver(["F %d %d %d " % c[:3] + " ".join("%x" % x for x in c[3] + c[4]) for c in cases])
    seen = set()
    for case, g in zip(cases, got):
        want = parse_rule(*case)
        assert tuple(int(v, 16) if k >= 3 else int(v) for k, v in enumerate(g[:len(want)])) == want, (case, want, g)
        seen.add(want[0])
    assert seen == {OK, INVALID}
