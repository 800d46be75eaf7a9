"""GPU tests of the decoder's integrity check (fpngb_set_decode_verify) at the edges of its four checksum kernels: the cases of
tests/checksum_edges.py, whose expected statuses come from zlib, through every decode entry point that takes them.  With the check
on every file gets its expected status and a failing file's output keeps its guard bytes; with it off clean files decode to the
same pixels and damaged fpng files as the reference decodes them (general files as zlib inflates them)."""
import struct
import zlib

import numpy as np
import pytest

import checksum_edges as ce
import pngwrite
from test_decode_device_gpu import to_device
from test_decode_ragged_gpu import pack_at

pytestmark = pytest.mark.gpu
GUARD = 0x5A


@pytest.fixture(autouse=True)
def _verify_off_after():
    yield
    import fpng_b200
    fpng_b200.set_decode_verify(False)


@pytest.fixture(scope="module")
def reference(oracle):
    """the reference where oracle/_ref was built, else the oracle (byte-identical decoder)"""
    import refreplay
    return refreplay.reference("Ref") if refreplay._live_available("Ref") else oracle


@pytest.fixture(scope="module")
def fpng(oracle, reference):
    """the fpng cases with the reference's decode (status, pixels at the file's channel count) of each"""
    cases = ce.fpng_cases(oracle)
    return [(c, reference.decode(c.png, ce.fpng_shape(c.png)[2])[:2]) for c in cases]


@pytest.fixture(scope="module")
def general():
    return ce.general_cases()


def need_free(gb):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * gb * 1e9:
        pytest.skip(f"needs {gb} GB of device memory and three times that free; {free / 1e9:.1f} GB free")


def test_fpng_host(gpu, fpng):
    """fpng_decode_memory: the uniform host path (its CRC grid from the file's own IDAT length)"""
    for c, (rst, rpx) in fpng:
        ch = ce.fpng_shape(c.png)[2]
        gpu.set_decode_verify(False)
        st, px = gpu.fpng_decode_memory(c.png, ch)[:2]
        assert st == rst and (px is None) == (rpx is None), c.name
        assert px is None or np.array_equal(px, rpx), c.name
        gpu.set_decode_verify(True)
        st2, px2 = gpu.fpng_decode_memory(c.png, ch)[:2]
        assert st2 == c.want, (c.name, st2, c.want)
        assert (px2 is None) if c.want else np.array_equal(px2, px), c.name


def run_packed(gpu, files, w, h, ch):
    """decode_packed_device (interleaved and planar, max_file_size = the largest file) and decode_batch_device of files of one
    shape into guard-filled outputs: [(statuses, pixels [n, h, w, ch])] per call"""
    import torch
    n = len(files)
    buf, offs = pack_at(files, np.random.RandomState(n), False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    mfs = max(len(f) for f in files)
    out = torch.full((n, h, w, ch), GUARD, dtype=torch.uint8, device="cuda")
    _, st = gpu.decode_packed_device(data, offsets, sizes, w, h, ch, ch, max_file_size=mfs, out=out)
    planar = torch.full((n, ch, h, w), GUARD, dtype=torch.uint8, device="cuda")
    _, st2 = gpu.decode_packed_device(data, offsets, sizes, w, h, ch, ch, max_file_size=mfs, out=planar.permute(0, 2, 3, 1))
    stride = (mfs + 16 + 15) // 16 * 16
    dev = torch.zeros((n, stride), dtype=torch.uint8, device="cuda")
    io, il = [], []
    for i, f in enumerate(files):
        dev[i, :len(f)] = torch.from_numpy(np.frombuffer(f, np.uint8).copy())
        info = gpu.get_info_ex(f)
        assert info[0] == 0
        io.append(info[4]); il.append(info[5])
    bout = torch.full((n, h, w, ch), GUARD, dtype=torch.uint8, device="cuda")
    _, st3 = gpu.decode_batch_device(dev, [len(f) for f in files], io, il, w, h, ch, ch, out=bout)
    torch.cuda.synchronize()
    return [(st.cpu().numpy(), out.cpu().numpy()), (st2.cpu().numpy(), planar.permute(0, 2, 3, 1).cpu().numpy()),
            (st3.cpu().numpy(), bout.cpu().numpy())]


def test_fpng_packed_and_batch(gpu, fpng):
    groups = {}
    for c, ref in fpng:
        groups.setdefault(ce.fpng_shape(c.png)[:3], []).append((c, ref))
    for (w, h, ch), group in groups.items():
        files = [c.png for c, _ in group]
        gpu.set_decode_verify(False)
        off = run_packed(gpu, files, w, h, ch)
        gpu.set_decode_verify(True)
        on = run_packed(gpu, files, w, h, ch)
        for k in range(3):
            for i, (c, (rst, rpx)) in enumerate(group):
                assert off[k][0][i] == rst, (c.name, k, off[k][0][i], rst)
                if rst == 0:
                    assert np.array_equal(off[k][1][i].reshape(-1), rpx), (c.name, k)
                assert on[k][0][i] == c.want, (c.name, k, on[k][0][i], c.want)
                if c.want:
                    assert (on[k][1][i] == GUARD).all(), (c.name, k)
                else:
                    assert np.array_equal(on[k][1][i], off[k][1][i]), (c.name, k)


def run_ragged(gpu, files, d, **flags):
    """one ragged call with every bound given (max_file_size = the largest file) into a guard-filled output: (statuses, out,
    out_offsets, info)"""
    import torch
    buf, offs = pack_at(files, np.random.RandomState(len(files)), False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    infos = [gpu.get_png_info(f, all_formats=True) for f in files]
    cap = sum((i[1] * i[2] * d + 15) // 16 * 16 for i in infos)
    out = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out[:cap], max_file_size=max(len(f) for f in files),
                                                      max_w=max(i[1] for i in infos), max_h=max(i[2] for i in infos), **flags)
    torch.cuda.synchronize()
    return st.cpu().numpy(), out.cpu().numpy(), oo.cpu().numpy(), info.cpu().numpy()


def check_ragged(gpu, cases, d, off_status, off_pixels, **flags):
    """cases: [Case]; off_status[i] / off_pixels[i] (or None: not compared) the expected result of file i with the check off"""
    files = [c.png for c in cases]
    gpu.set_decode_verify(False)
    st0, out0, oo0, info = run_ragged(gpu, files, d, **flags)
    gpu.set_decode_verify(True)
    st1, out1, oo1, _ = run_ragged(gpu, files, d, **flags)
    assert np.array_equal(oo0, oo1)
    for i, c in enumerate(cases):
        size = int(info[i][1]) * int(info[i][2]) * d
        o = int(oo1[i])
        assert st0[i] == off_status[i], (c.name, flags, st0[i], off_status[i])
        if st0[i] == 0 and off_pixels[i] is not None:
            assert np.array_equal(out0[o:o + size], off_pixels[i].reshape(-1)), (c.name, flags)
        assert st1[i] == c.want, (c.name, flags, st1[i], c.want)
        if c.want:
            assert (out1[o:o + size] == GUARD).all(), (c.name, flags)
        else:
            assert np.array_equal(out1[o:o + size], out0[o:o + size]), (c.name, flags)


def test_fpng_ragged(gpu, fpng, reference):
    """decode_packed_ragged_device over every fpng case in one call, plain, any_png and all_formats"""
    cases = [c for c, _ in fpng]
    ref4 = [reference.decode(c.png, 4)[:2] for c in cases]
    for flags in ({}, dict(any_png=True), dict(any_png=True, all_formats=True)):
        check_ragged(gpu, cases, 4, [r[0] for r in ref4], [r[1] for r in ref4], **flags)


def test_general_ragged(gpu, general, fpng):
    """the general cases with a few clean fpng files, through the any_png (8-bit files) and all_formats (all) ragged decodes"""
    extra = [(c, ref) for c, ref in fpng if c.name.startswith("crc_tail")][:4]
    for d in (3, 4):
        for flags, kinds in ((dict(any_png=True), ("png",)), (dict(any_png=True, all_formats=True), ("png", "ext"))):
            cases = [c for c in general if c.kind in kinds]
            want_off = [c.want_off for c in cases]
            px = [pngwrite.expand(c.pixels, d) if c.kind == "png" and "damage" not in c.name else None for c in cases]
            for c, (rst, _) in extra:
                cases.append(c)
                want_off.append(rst)
                px.append(None)
            check_ragged(gpu, cases, d, want_off, px, **flags)


def test_big_file_past_2_32_bits(gpu):
    """RGBA noise of 16384 x 8448 (stored blocks, IDAT 553 MB > 2^29 bytes): the CRC's shifts need exponent bits >= 32.  With the
    check on the clean file decodes, a flipped byte at each of
    checksum_edges.big_damage_spots gives 4 and a flipped Adler-32 bit (CRC rewritten) gives 102, on the host path and in one packed
    call with max_file_size the largest file.  The encoder's CRC field agrees with zlib."""
    import torch
    need_free(3)
    torch.cuda.reset_peak_memory_stats()
    W, H, C = ce.BIG_W, ce.BIG_H, ce.BIG_C
    g = torch.Generator(device="cuda").manual_seed(5)
    img = torch.randint(0, 256, (1, H, W, C), dtype=torch.uint8, device="cuda", generator=g)
    out, sizes = gpu.encode_batch_device(img)
    torch.cuda.synchronize()
    png = out[0, :int(sizes[0].item()) & 0xFFFFFFFF].cpu().numpy().tobytes()
    del out
    pixels = img[0].cpu().numpy().reshape(-1)
    w, h, ch, m0, L, ofs, n = ce.fpng_shape(png)
    assert (w, h, ch, m0) == (W, H, C, ce.FPNG_MSG_START) and L - m0 == ce.big_message_len() > 1 << 29
    # the encoder's stored path runs the same CRC kernel: its CRC field is compared with zlib's at the end, and the decode checks
    # below run on the file with zlib's CRC, so that they test the verify path on their own
    encoder_crc = struct.unpack(">I", png[L:L + 4])[0]
    crc = zlib.crc32(png[m0:L]) & 0xFFFFFFFF
    png = png[:L] + struct.pack(">I", crc) + png[L + 4:]
    gpu.set_decode_verify(True)
    st, px = gpu.fpng_decode_memory(png, C)[:2]
    assert st == 0 and np.array_equal(px, pixels)
    del px
    for at in ce.big_damage_spots():
        b = bytearray(png)
        b[at] ^= 0x08
        assert gpu.fpng_decode_memory(bytes(b), C)[0] == ce.CRC, at
    b = bytearray(png)
    b[L - 1] ^= 0x01                                                             # the Adler-32's last byte
    b[L:L + 4] = struct.pack(">I", zlib.crc32(bytes(b[m0:L])) & 0xFFFFFFFF)
    bad_adler = bytes(b)
    del b
    assert gpu.fpng_decode_memory(bad_adler, C)[0] == ce.ADLER
    # one packed call: the clean file, the Adler-damaged one and the first damage spot
    first = bytearray(png)
    first[ce.big_damage_spots()[0]] ^= 0x08
    files = [png, bad_adler, bytes(first)]
    del first
    buf, offs = pack_at(files, np.random.RandomState(0), True)
    data, offsets, szs = to_device(buf, offs, [len(f) for f in files])
    del buf
    o = torch.full((3, H, W, C), GUARD, dtype=torch.uint8, device="cuda")
    _, st = gpu.decode_packed_device(data, offsets, szs, W, H, C, C, max_file_size=max(len(f) for f in files), out=o)
    assert st.cpu().tolist() == [0, ce.ADLER, ce.CRC]
    assert torch.equal(o[0], img[0]) and bool((o[1:] == GUARD).all())
    assert encoder_crc == crc
    print(f"big file: IDAT {n} bytes, torch peak {torch.cuda.max_memory_allocated() / 1e9:.2f} GB")
