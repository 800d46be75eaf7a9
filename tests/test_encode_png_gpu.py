"""GPU tests of encode_png_device / fpngb_encode_png_ragged_device: gray, gray+alpha and 16-bit device images encoded to PNG.
Every new file must equal the oracle's (oracle/png_encode_oracle.c) byte for byte, the fpng files of a mixed list must equal
encode_ragged_device's, and the files must decode on the GPU through the all-formats decoder."""
import ctypes as C
import threading

import numpy as np
import pytest

import imagegen
import pngenc_workloads as pw

pytestmark = pytest.mark.gpu

INVALID_ARG, TOO_SMALL, ALIGNMENT = 1, 2, 5
GUARD = 0xA5


@pytest.fixture(scope="module")
def env():
    import fpng_b200
    from oracle.pngenc_oracle import PngEncodeOracle
    fpng_b200.fpng_init(0)
    return fpng_b200, PngEncodeOracle()


def dev(img):
    import torch
    return torch.from_numpy(np.ascontiguousarray(img)).cuda()


def files(out, offsets, sizes):
    import torch
    torch.cuda.synchronize()
    data, ofs, sz = out.cpu().numpy(), offsets.cpu().numpy(), sizes.cpu().numpy().astype(np.int64)
    return [data[ofs[i]:ofs[i] + sz[i]].tobytes() for i in range(len(sz))]


def check_against_oracle(fp, o, imgs, flags=0, views=None):
    out, offsets, sizes = fp.encode_png_device(views if views is not None else [dev(i) for i in imgs], flags)
    got = files(out, offsets, sizes)
    shapes = [(i.shape[0], i.shape[1], i.shape[2], 8 * i.dtype.itemsize) for i in imgs]
    assert offsets.cpu().numpy().tolist() == fp.png_slot_offsets(shapes).tolist()
    for k, img in enumerate(imgs):
        assert got[k] == o.png_encode(img, flags), (k, img.shape, img.dtype, flags)
    return out, offsets, sizes


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_corpus_matches_oracle(env, flags):
    fp, o = env
    check_against_oracle(fp, o, [img for _, img in pw.corpus()], flags)


@pytest.mark.parametrize("name", list(pw.WORKLOADS))
def test_workloads_match_oracle(env, name):
    fp, o = env
    check_against_oracle(fp, o, pw.workload(name, 4))


def test_layouts(env):
    """crops at odd pitches, planar CHW through permute, and expand with a zero row stride read in place"""
    import torch
    fp, o = env
    rng = np.random.default_rng(3)
    imgs, views = [], []
    for c, dt in ((1, np.uint8), (2, np.uint8), (1, np.uint16), (2, np.uint16), (3, np.uint16), (4, np.uint16)):
        canvas = (rng.integers(0, 4, (21, 37, c)) * 4000).astype(dt) if dt == np.uint16 else rng.integers(0, 4, (21, 37, c)).astype(dt)
        t = dev(canvas)
        crop = t[2:19, 3:30]                                          # row pitch of 37 pixels: odd for every element size
        imgs.append(canvas[2:19, 3:30]); views.append(crop)
        chw = dev(np.ascontiguousarray(canvas.transpose(2, 0, 1)))
        imgs.append(canvas); views.append(chw.permute(1, 2, 0))
        row = dev(canvas[:1])
        imgs.append(np.repeat(canvas[:1], 9, axis=0)); views.append(row.expand(9, -1, -1))
    assert not views[0].is_contiguous() and views[2].stride()[0] == 0
    check_against_oracle(fp, o, imgs, views=views)
    torch.cuda.synchronize()


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_mixed_with_fpng_images(env, flags):
    """uint8 RGB / RGBA images in the same call are fpng files, byte-identical to encode_ragged_device's"""
    fp, o = env
    rgb = [imagegen.make("g1", w, h, c, s).reshape(h, w, c) for s, (h, w, c) in enumerate([(17, 33, 3), (40, 512, 4), (5, 1, 3)])]
    new = [img for _, img in pw.corpus()[::9]]
    mixed = [rgb[0]] + new[:3] + [rgb[1]] + new[3:] + [rgb[2]]
    got = files(*fp.encode_png_device([dev(i) for i in mixed], flags))
    ref = files(*fp.encode_ragged_device([dev(i) for i in rgb], flags))
    assert [got[0], got[4], got[-1]] == ref
    for k, img in enumerate(new):
        assert got[1 + k + (k >= 3)] == o.png_encode(img, flags)


def test_neighbours_do_not_matter(env):
    fp, o = env
    corpus = [img for _, img in pw.corpus()]
    alone = [files(*fp.encode_png_device([dev(img)]))[0] for img in corpus[::11]]
    together = files(*fp.encode_png_device([dev(img) for img in corpus[::-1]]))[::-1][::11]
    assert alone == together


def test_round_trip_all_formats_decode(env):
    """Decoded to 4 channels by the all-formats decoder: the uint8 output holds each sample's high byte, a float32 output with
    scale 257 rounds back to every 16-bit sample (gray is replicated to RGB; alpha the file lacks is not compared)."""
    import torch
    fp, o = env
    imgs = [img for _, img in pw.corpus()][::3] + pw.workload("E2", 2)
    out, offsets, sizes = fp.encode_png_device([dev(i) for i in imgs])
    px, pofs, info, status = fp.decode_packed_ragged_device(out, offsets[:-1].contiguous(), sizes, 4, any_png=True, all_formats=True)
    fx, fofs, _, fstatus = fp.decode_packed_ragged_device(out, offsets[:-1].contiguous(), sizes, 4, any_png=True, all_formats=True,
                                                          dtype=torch.float32, scale=257.0)
    torch.cuda.synchronize()
    assert not status.any().item() and not fstatus.any().item()
    px, pofs, fx, fofs = px.cpu().numpy(), pofs.cpu().numpy(), fx.cpu().numpy(), fofs.cpu().numpy()
    for k, img in enumerate(imgs):
        h, w, c = img.shape
        cols = [[0, 0, 0], [0, 0, 0, 1], [0, 1, 2], [0, 1, 2, 3]][c - 1]
        u8 = px.view(np.uint8)[pofs[k]:pofs[k] + 4 * h * w].reshape(h, w, 4)[..., :len(cols)]
        hi = (img >> 8).astype(np.uint8) if img.dtype == np.uint16 else img
        assert np.array_equal(u8, hi[..., cols]), (k, img.shape, img.dtype)
        f = fx.view(np.uint8)[fofs[k]:fofs[k] + 16 * h * w].view(np.float32).reshape(h, w, 4)[..., :len(cols)]
        want = img.astype(np.int64) if img.dtype == np.uint16 else img.astype(np.int64) * 257
        assert np.array_equal(np.round(f).astype(np.int64), want[..., cols]), (k, img.shape, img.dtype)


def test_rejections_enqueue_nothing(env):
    import torch
    fp, o = env
    from fpng_b200._lib import lib
    L = lib()
    img = dev(np.zeros((4, 5, 1), np.uint16))
    out = torch.full((4096,), GUARD, dtype=torch.uint8, device="cuda")
    offs = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((1,), -7, dtype=torch.int32, device="cuda")

    def call(dims, flags=0, n=1, ptr=None, strides=None, cap=4096, out_ptr=None):
        ptrs = np.array([img.data_ptr() if ptr is None else ptr], np.uint64)
        d = np.array(dims, np.uint32)
        st = None if strides is None else np.array(strides, np.uint64).ctypes.data_as(C.c_void_p)
        return L.fpngb_encode_png_ragged_device(n, ptrs.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p), st, flags,
                                                out.data_ptr() if out_ptr is None else out_ptr, cap, offs.data_ptr(), sizes.data_ptr(), None)

    torch.cuda.synchronize()
    before = fp.launch_count()
    assert call([5, 4, 1, 12]) == INVALID_ARG                        # depth
    assert call([5, 4, 0, 16]) == INVALID_ARG                        # channels
    assert call([5, 4, 5, 16]) == INVALID_ARG
    assert call([5, 4, 1, 16], flags=4) == INVALID_ARG               # unknown flag bit
    assert call([5, 4, 1, 16], n=0) == INVALID_ARG
    assert call([5, 4, 1, 16], ptr=0) == INVALID_ARG
    assert call([1 << 24, 40, 4, 16]) == INVALID_ARG                 # slot bound above 2^31 - 1
    assert call([5, 0, 1, 16]) == INVALID_ARG
    assert call([5, 4, 1, 16], cap=16) == TOO_SMALL
    assert call([5, 4, 1, 16], out_ptr=out.data_ptr() + 8) == ALIGNMENT
    assert call([5, 4, 1, 16], ptr=img.data_ptr() + 1) == ALIGNMENT   # odd address of 16-bit samples
    assert call([5, 4, 2, 16], strides=[20, 4, 3]) == ALIGNMENT       # odd channel stride
    assert call([5, 4, 2, 8], strides=[10, 3, 1]) == INVALID_ARG     # neither interleaved nor planar
    torch.cuda.synchronize()
    assert fp.launch_count() == before
    assert (out == GUARD).all().item() and (offs == -7).all().item() and (sizes == -7).all().item()
    with pytest.raises(ValueError):
        fp.encode_png_device([dev(np.zeros((2, 2, 1), np.int16))])


def test_thousands_of_files_on_two_streams(env):
    import torch
    fp, o = env
    rng = np.random.default_rng(11)
    fmts = ((1, np.uint8), (2, np.uint8), (1, np.uint16), (2, np.uint16), (3, np.uint16), (4, np.uint16))
    lists = []
    for s in range(2):
        imgs = []
        for k in range(1500):
            c, dt = fmts[(k + s) % 6]
            h, w = int(rng.integers(1, 24)), int(rng.integers(1, 40))
            top = 4 if k % 3 else (256 if dt == np.uint8 else 65536)
            imgs.append(rng.integers(0, top, (h, w, c)).astype(dt))
        lists.append(imgs)
    streams = [torch.cuda.Stream() for _ in range(2)]
    tens = [[dev(i) for i in imgs] for imgs in lists]
    torch.cuda.synchronize()
    results = [None, None]

    def run(s):
        with torch.cuda.stream(streams[s]):
            results[s] = fp.encode_png_device(tens[s])

    th = [threading.Thread(target=run, args=(s,)) for s in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    for s in range(2):
        got = files(*results[s])
        for k, img in enumerate(lists[s]):
            assert got[k] == o.png_encode(img), (s, k, img.shape, img.dtype)
