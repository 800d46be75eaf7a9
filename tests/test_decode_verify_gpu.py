"""GPU tests of the decoder's opt-in integrity check (fpngb_set_decode_verify): the IDAT CRC-32 and the zlib Adler-32 checked on
the GPU in every decode entry point.  Damaged files are built here from clean ones.  With the switch off every case decodes as
the reference decodes it; with it on the statuses follow the documented precedence (CRC, then the stream, then Adler-32), a
failing file's output stays untouched, and the clean files around it decode to the same bytes as with the switch off."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import imagegen
import streamgen
from common import golden_vectors, with_text_chunk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CRC, NOT_FPNG, ADLER = 4, 1, 102
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


def idat(gpu, png):
    st, w, h, c, ofs, n = gpu.get_info_ex(png)
    assert st == 0
    return ofs, n


def with_crc(png, ofs, n):
    b = bytearray(png)
    b[ofs + 8 + n:ofs + 12 + n] = struct.pack(">I", zlib.crc32(bytes(b[ofs + 4:ofs + 8 + n])) & 0xFFFFFFFF)
    return bytes(b)


def damaged(gpu, oracle):
    """[(name, file, status with the switch on)] in the order of the issue's cases"""
    img = imagegen.make("g1", 67, 19, 3, 3)
    png = oracle.encode(img, 67, 19, 3, 0)
    ofs, n = idat(gpu, png)
    out = []
    b = bytearray(png); b[ofs + 8 + n] ^= 0x01
    out.append(("crc_field", bytes(b), CRC))
    b = bytearray(png); b[ofs + 8 + n // 2] ^= 0x10
    out.append(("data_byte", bytes(b), CRC))
    b = bytearray(png); b[ofs + 8 + n - 2] ^= 0x40
    out.append(("adler_rewritten", with_crc(bytes(b), ofs, n), ADLER))
    stored = oracle.encode(img, 67, 19, 3, 2)
    so, sn = idat(gpu, stored)
    b = bytearray(stored); b[so + 8 + 2 + 5 + 500] ^= 0x04                   # a pixel byte of the first stored block (not a filter byte)
    out.append(("stored_pixel", with_crc(bytes(b), so, sn), ADLER))
    name, f, chans, ok, dev, data = [c for c in streamgen.cases() if c[0] == "flat286_c3"][0]
    st, w, h, c, zo, zn = gpu.get_info_ex(f)
    z = f[zo + 8:zo + 8 + zn]
    other = bytearray(data); other[len(other) // 2] ^= 0x01
    out.append(("streamgen_adler", streamgen.png_file(w, h, chans, streamgen.zlib_stream(z[2:-4], bytes(other))), ADLER))
    b = bytearray(png); b[ofs + 8 + n - 1] ^= 0x01                           # Adler wrong, CRC left as it was
    out.append(("crc_and_adler", bytes(b), CRC))
    b = bytearray(png); b[ofs + 8] = 0x00                                    # zlib header broken, CRC left as it was
    out.append(("crc_and_stream", bytes(b), CRC))
    return out


def clean_files(gpu, oracle):
    """clean files of one shape (67 x 19 RGB) in 1-pass, 2-pass and stored modes, GPU- and oracle-written"""
    out = []
    for k, flags in enumerate((0, 1, 2)):
        img = imagegen.make("g1", 67, 19, 3, 10 + k)
        out.append(oracle.encode(img, 67, 19, 3, flags))
        ok, g = gpu.fpng_encode_image_to_memory(img, 67, 19, 3, flags)
        assert ok
        out.append(g)
    return out


def test_host_entry_points(gpu, oracle, reference):
    cases = damaged(gpu, oracle)
    clean = clean_files(gpu, oracle)
    for d in (3, 4):
        for name, f, want in cases:
            rst, rpx = reference.decode(f, d)[:2]
            gpu.set_decode_verify(False)
            st, px = gpu.fpng_decode_memory(f, d)[:2]
            assert st == rst, name
            assert (px is None) == (rpx is None) and (px is None or np.array_equal(px, rpx)), name
            gpu.set_decode_verify(True)
            st, px = gpu.fpng_decode_memory(f, d)[:2]
            assert (st, px) == (want, None), name
        gpu.set_decode_verify(True)
        files = []
        for f in clean:
            files.append(f)
        files += [f for _, f, _ in cases if gpu.get_info_ex(f)[1:4] == (67, 19, 3)]
        res = gpu.decode_files(files, d)
        wants = [0] * len(clean) + [w for _, f, w in cases if gpu.get_info_ex(f)[1:4] == (67, 19, 3)]
        assert [r[0] for r in res] == wants
        gpu.set_decode_verify(False)
        off = gpu.decode_files(files, d)
        for r, o, w in zip(res, off, wants):
            if w == 0:
                assert o[0] == 0 and np.array_equal(r[1], o[1])


def test_alignments_and_golden_clean(gpu, oracle):
    """clean files with IDAT at every start alignment, example.png and the golden vectors: status 0, same bytes as switch off"""
    img = imagegen.make("g1", 131, 37, 4, 5)
    png = oracle.encode(img, 131, 37, 4, 0)
    files = [with_text_chunk(png, k) for k in range(4)]
    with open(os.path.join(ROOT, "tests", "golden", "example.png"), "rb") as fh:
        files.append(fh.read())
    for v in golden_vectors():
        if "png_hex" in v:
            files.append(bytes.fromhex(v["png_hex"]))
    for f in files:
        for d in (3, 4):
            gpu.set_decode_verify(False)
            o = gpu.fpng_decode_memory(f, d)
            gpu.set_decode_verify(True)
            r = gpu.fpng_decode_memory(f, d)
            assert r[0] == o[0]
            if o[0] == 0:
                assert np.array_equal(r[1], o[1])
    # a damaged byte at every alignment is caught
    for k in range(4):
        f = with_text_chunk(png, k)
        ofs, n = idat(gpu, f)
        for at in (0, 1, n // 2, n - 1):
            b = bytearray(f); b[ofs + 8 + at] ^= 0x80
            assert gpu.fpng_decode_memory(bytes(b), 4)[0] == CRC, (k, at)


def packed(files):
    offs, at = [], 0
    for f in files:
        at = (at + 15) // 16 * 16
        offs.append(at)
        at += len(f)
    buf = np.zeros(at + 16, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(bytes(f), np.uint8)
    return buf, offs


def test_device_entry_points(gpu, oracle):
    import torch
    cases = [c for c in damaged(gpu, oracle) if gpu.get_info_ex(c[1])[1:4] == (67, 19, 3)]
    clean = clean_files(gpu, oracle)
    files = clean[:3] + [f for _, f, _ in cases] + clean[3:]
    wants = [0] * 3 + [w for _, _, w in cases] + [0] * len(clean[3:])
    n = len(files)
    buf, offs = packed(files)
    data = torch.from_numpy(buf).cuda()
    offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
    sizes = torch.tensor([len(f) for f in files], dtype=torch.int32, device="cuda")
    mfs = max(len(f) for f in files)
    for d in (3, 4):
        res = {}
        for on in (False, True):
            gpu.set_decode_verify(on)
            out = torch.full((n, 19, 67, d), GUARD, dtype=torch.uint8, device="cuda")
            _, st = gpu.decode_packed_device(data, offsets, sizes, 67, 19, 3, d, max_file_size=mfs, out=out)
            planar = torch.full((n, d, 19, 67), GUARD, dtype=torch.uint8, device="cuda")
            _, st2 = gpu.decode_packed_device(data, offsets, sizes, 67, 19, 3, d, max_file_size=mfs, out=planar.permute(0, 2, 3, 1))
            slot = (67 * 19 * d + 15) // 16 * 16
            rout, roffs, info, rst = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=torch.full((n * slot + 64,), GUARD, dtype=torch.uint8, device="cuda"),
                                                                     max_file_size=mfs, max_w=67, max_h=19)
            stride = (max(len(f) for f in files) + 16 + 15) // 16 * 16
            dev = torch.zeros((n, stride), dtype=torch.uint8, device="cuda")
            io, il = [], []
            for i, f in enumerate(files):
                dev[i, :len(f)] = torch.from_numpy(np.frombuffer(bytes(f), np.uint8).copy())
                s, *_rest = gpu.get_info_ex(f)
                io.append(_rest[3]); il.append(_rest[4])
            bout = torch.full((n, 19, 67, d), GUARD, dtype=torch.uint8, device="cuda")
            _, st3 = gpu.decode_batch_device(dev, [len(f) for f in files], io, il, 67, 19, 3, d, out=bout)
            torch.cuda.synchronize()
            res[on] = (out.cpu().numpy(), st.cpu().numpy(), planar.cpu().numpy(), st2.cpu().numpy(), rout.cpu().numpy(), rst.cpu().numpy(),
                       bout.cpu().numpy(), st3.cpu().numpy(), roffs.cpu().numpy())
        off, on = res[False], res[True]
        for k in (1, 3, 5, 7):
            assert on[k].tolist() == wants, k
        for i, w in enumerate(wants):
            for k in (0, 2, 6):
                if w:
                    assert (on[k][i] == GUARD).all()
                else:
                    assert np.array_equal(on[k][i], off[k][i])
            o = int(on[8][i]); size = 67 * 19 * d
            if w:
                assert (on[4][o:o + size] == GUARD).all()
            else:
                assert np.array_equal(on[4][o:o + size], off[4][o:o + size])


def test_ragged_mix_and_launches(gpu, oracle):
    import torch
    rs = np.random.RandomState(3)
    files, wants = [], []
    for i in range(24):
        w, h, c = int(rs.choice([1, 7, 64, 333, 1920])), int(rs.randint(1, 40)), int(rs.choice([3, 4]))
        png = oracle.encode(imagegen.make("g1", w, h, c, i), w, h, c, int(rs.choice([0, 1, 2])))
        if i % 3 == 2:
            ofs, n = idat(gpu, png)
            b = bytearray(png); b[ofs + 8 + int(rs.randint(0, n))] ^= 0x20
            png, want = bytes(b), CRC
        else:
            want = 0
        files.append(png); wants.append(want)
    buf, offs = packed(files)
    data = torch.from_numpy(buf).cuda()
    offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
    sizes = torch.tensor([len(f) for f in files], dtype=torch.int32, device="cuda")
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=1920, max_h=40)
    cap = sum((gpu.get_info_ex(f)[1] * gpu.get_info_ex(f)[2] * 4 + 15) // 16 * 16 for f in files)
    res = {}
    for on in (False, True):
        gpu.set_decode_verify(on)
        out = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        before = gpu.launch_count()
        r = gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out, **bounds)
        res[on] = (gpu.launch_count() - before, r[0].cpu().numpy(), r[1].cpu().numpy(), r[3].cpu().numpy())
    assert res[True][0] == res[False][0] + 2
    assert res[True][3].tolist() == wants
    assert all(s == 0 for s, w in zip(res[False][3].tolist(), wants) if w == 0)
    for i, (f, w) in enumerate(zip(files, wants)):
        o = int(res[True][2][i]); size = gpu.get_info_ex(f)[1] * gpu.get_info_ex(f)[2] * 4
        if w:
            assert (res[True][1][o:o + size] == GUARD).all()
        else:
            assert np.array_equal(res[True][1][o:o + size], res[False][1][o:o + size])


def test_no_host_synchronisation(gpu, oracle):
    """with the switch on, the packed and ragged calls enqueue behind a long-running kernel without waiting for it"""
    import time

    import torch
    png = oracle.encode(imagegen.make("g1", 64, 32, 3, 0), 64, 32, 3, 0)
    buf, offs = packed([png] * 8)
    data = torch.from_numpy(buf).cuda()
    offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
    sizes = torch.tensor([len(png)] * 8, dtype=torch.int32, device="cuda")
    gpu.set_decode_verify(True)
    gpu.decode_packed_device(data, offsets, sizes, 64, 32, 3, 3, max_file_size=len(png))          # warm
    gpu.decode_packed_ragged_device(data, offsets, sizes, 3, out=torch.empty(8 * 64 * 32 * 3 + 64, dtype=torch.uint8, device="cuda"),
                                    max_file_size=len(png), max_w=64, max_h=32)
    out = torch.empty(8 * 64 * 32 * 3 + 64, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))                                                                    # ~1 s of GPU time on the stream
    t0 = time.perf_counter()
    _, st = gpu.decode_packed_device(data, offsets, sizes, 64, 32, 3, 3, max_file_size=len(png))
    r = gpu.decode_packed_ragged_device(data, offsets, sizes, 3, out=out, max_file_size=len(png), max_w=64, max_h=32)
    enq = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert enq < 0.2, enq
    assert st.cpu().tolist() == [0] * 8 and r[3].cpu().tolist() == [0] * 8


def test_large_file_multi_cta(gpu):
    """3840 x 2160 RGBA: the CRC runs over many CTAs; a damaged first, middle and last IDAT byte is caught, the clean file decodes"""
    import torch
    img = imagegen.make("g1", 3840, 2160, 4, 1)
    ok, png = gpu.fpng_encode_image_to_memory(img, 3840, 2160, 4, 0)
    assert ok
    ofs, n = idat(gpu, png)
    files = [png]
    for at in (0, n // 2, n - 1):
        b = bytearray(png); b[ofs + 8 + at] ^= 0x01
        files.append(bytes(b))
    buf, offs = packed(files)
    data = torch.from_numpy(buf).cuda()
    offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
    sizes = torch.tensor([len(f) for f in files], dtype=torch.int32, device="cuda")
    gpu.set_decode_verify(True)
    out = torch.full((4, 2160, 3840, 4), GUARD, dtype=torch.uint8, device="cuda")
    _, st = gpu.decode_packed_device(data, offsets, sizes, 3840, 2160, 4, 4, max_file_size=max(map(len, files)), out=out)
    assert st.cpu().tolist() == [0, CRC, CRC, CRC]
    assert np.array_equal(out[0].cpu().numpy().reshape(-1), img.reshape(-1))
    assert bool((out[1:] == GUARD).all())


def test_cpp_no_fallback(tmp_path):
    """fpng::fpng_decode_memory returns 102 and 4 with the switch on and a fallback registered, without calling it"""
    from fpng_b200 import _build
    lib = _build.build()
    exe = str(tmp_path / "verify_test")
    subprocess.check_call(["g++", "-O2", "-std=c++11", os.path.join(ROOT, "tests", "cpp", "verify_test.cpp"), "-I" + os.path.join(ROOT, "include"),
                           "-L" + os.path.dirname(lib), "-lfpng_b200", "-Wl,-rpath," + os.path.dirname(lib), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "0 failures" in out.stdout
