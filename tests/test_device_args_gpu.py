"""GPU tests of the Python device functions' checks on the tensors a caller passes them (out, sizes, status): each refuses a
tensor that is too small, of the wrong dtype, on the host or in an unsupported layout with ValueError before anything is
enqueued, and decode_batch_device never waits on the host for an earlier call's upload."""
import time

import numpy as np
import pytest

import imagegen
from test_decode_device_gpu import packed_device

pytestmark = pytest.mark.gpu

W, H, C, N = 37, 11, 3, 4


@pytest.fixture(scope="module")
def case(gpu):
    import torch
    imgs = torch.from_numpy(np.stack([imagegen.make("g1", W, H, C, i) for i in range(N)]).reshape(N, H, W, C)).cuda()
    out, sizes = gpu.encode_batch_device(imgs)
    sz = sizes.cpu().numpy()
    files = [out[i, :sz[i]].cpu().numpy().tobytes() for i in range(N)]
    return imgs, files


def refused(gpu, call):
    before = gpu.launch_count()
    with pytest.raises(ValueError):
        call()
    assert gpu.launch_count() == before, "a refused call launched kernels"


def test_encode_batch_device_checks_out_and_sizes(gpu, case):
    import torch
    imgs, _ = case
    row = (gpu.max_encoded_size(W, H, C) + 15) // 16 * 16
    good_out = torch.empty((N, row), dtype=torch.uint8, device="cuda")
    good_sizes = torch.empty((N,), dtype=torch.int32, device="cuda")
    for out in (torch.empty((N - 1, row), dtype=torch.uint8, device="cuda"),                # too few rows
                torch.empty((N, gpu.max_encoded_size(W, H, C) - 1), dtype=torch.uint8, device="cuda"),   # rows too short
                torch.empty((N, row), dtype=torch.int8, device="cuda"),                     # wrong dtype
                torch.empty((row, N), dtype=torch.uint8, device="cuda").t(),                # rows not contiguous
                torch.empty((N * row,), dtype=torch.uint8, device="cuda"),                  # not [n, row]
                torch.empty((N, row), dtype=torch.uint8)):                                  # on the host
        refused(gpu, lambda: gpu.encode_batch_device(imgs, out=out, sizes=good_sizes))
    for sizes in (torch.empty((N - 1,), dtype=torch.int32, device="cuda"),
                  torch.empty((N,), dtype=torch.int64, device="cuda"),
                  torch.empty((N, 2), dtype=torch.int32, device="cuda")[:, 0],
                  torch.empty((N,), dtype=torch.int32)):
        refused(gpu, lambda: gpu.encode_batch_device(imgs, out=good_out, sizes=sizes))
    refused(gpu, lambda: gpu.encode_batch_device(imgs.float(), out=good_out, sizes=good_sizes[:N - 1], scale=1.0))
    o, s = gpu.encode_batch_device(imgs, out=good_out, sizes=good_sizes)                    # the same tensors, accepted
    assert o.data_ptr() == good_out.data_ptr() and s.data_ptr() == good_sizes.data_ptr()


@pytest.mark.parametrize("packed", [False, True])
def test_decode_device_checks_out_and_status(gpu, case, packed):
    import torch
    _, files = case
    if packed:
        data, offsets, sizes = packed_device(files)
        call = lambda **kw: gpu.decode_packed_device(data, offsets, sizes, W, H, C, C, **kw)   # noqa: E731
    else:
        t, _, fs, fo, fl, *_ = gpu.pack_files_for_device(files, "cuda")
        call = lambda **kw: gpu.decode_batch_device(t, fs, fo, fl, W, H, C, C, **kw)           # noqa: E731
    px = N * H * W * C
    good_status = torch.empty((N,), dtype=torch.int32, device="cuda")
    for kw in (dict(out=torch.empty((px - 1,), dtype=torch.uint8, device="cuda")),           # too small (the overrun of old)
               dict(out=torch.empty((N - 1, H, W, C), dtype=torch.uint8, device="cuda")),
               dict(out=torch.empty((N, H, W, C), dtype=torch.float32, device="cuda")[:N - 1], dtype=torch.float32),
               dict(out=torch.empty((N, H, W, C), dtype=torch.int32, device="cuda")),        # no such output dtype
               dict(out=torch.empty((N, H, W, C), dtype=torch.uint8, device="cuda"), dtype=torch.float16),
               dict(out=torch.empty((N, H, W, C + 1), dtype=torch.uint8, device="cuda")[..., :C]),   # not interleaved
               dict(out=torch.empty((N, H, 2 * W, C), dtype=torch.uint8, device="cuda")[:, :, ::2][:, :, :W - 1]),   # shape
               dict(out=torch.empty((N, H, W, C), dtype=torch.uint8)),                       # on the host
               dict(status=torch.empty((N - 1,), dtype=torch.int32, device="cuda")),
               dict(status=torch.empty((N,), dtype=torch.int64, device="cuda")),
               dict(status=torch.empty((N, 2), dtype=torch.int32, device="cuda")[:, 1]),
               dict(status=torch.empty((N,), dtype=torch.int32))):
        kw.setdefault("status", good_status)
        refused(gpu, lambda: call(**kw))
    out = torch.empty((px,), dtype=torch.uint8, device="cuda")                             # a flat out of the exact size is fine
    _, st = call(out=out, status=good_status)
    assert int(st.abs().sum()) == 0
    want = np.stack([np.frombuffer(gpu.fpng_decode_memory(f, C)[1].tobytes(), np.uint8) for f in files]).reshape(-1)
    assert np.array_equal(out.cpu().numpy(), want)


def test_ragged_and_compact_check_out(gpu, case):
    import torch
    imgs, files = case
    views = [imgs[i] for i in range(N)]
    for out in (torch.empty((1 << 16,), dtype=torch.int8, device="cuda"),
                torch.empty((2, 1 << 16), dtype=torch.uint8, device="cuda")[:, 0],
                torch.empty((1 << 16,), dtype=torch.uint8)):
        refused(gpu, lambda: gpu.encode_ragged_device(views, 0, out=out))
    data, offsets, sizes = packed_device(files)
    bounds = dict(max_file_size=max(map(len, files)), max_w=W, max_h=H)
    for kw in (dict(out=torch.empty((1 << 16,), dtype=torch.float32, device="cuda"), dtype=torch.float16),
               dict(out=torch.empty((2, 1 << 16), dtype=torch.uint8, device="cuda")[:, 0]),
               dict(out=torch.empty((1 << 16,), dtype=torch.uint8))):
        refused(gpu, lambda: gpu.decode_packed_ragged_device(data, offsets, sizes, C, **bounds, **kw))
    for out in (torch.empty((1 << 16,), dtype=torch.int32, device="cuda"), torch.empty((1 << 16,), dtype=torch.uint8)):
        refused(gpu, lambda: gpu.compact_packed_device(data, offsets, sizes, out=out))


def test_decode_batch_device_does_not_wait_for_an_earlier_upload(gpu, case):
    """a decode call on stream b while the previous call's FileDesc upload still waits on stream a behind ~0.5 s of GPU work"""
    import torch
    _, files = case
    t, _, fs, fo, fl, *_ = gpu.pack_files_for_device(files, "cuda")
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [torch.empty((N, H, W, C), dtype=torch.uint8, device="cuda") for _ in range(2)]
    with torch.cuda.stream(a):                                  # workspace and two staging slots reserved before the timed calls
        torch.cuda._sleep(1 << 26)
        gpu.decode_batch_device(t, fs, fo, fl, W, H, C, C, out=outs[0])
    with torch.cuda.stream(b):
        gpu.decode_batch_device(t, fs, fo, fl, W, H, C, C, out=outs[1])
    torch.cuda.synchronize()
    for o in outs:
        o.fill_(0)
    with torch.cuda.stream(a):
        torch.cuda._sleep(1 << 30)
        _, st_a = gpu.decode_batch_device(t, fs, fo, fl, W, H, C, C, out=outs[0])
    t0 = time.perf_counter()
    with torch.cuda.stream(b):
        _, st_b = gpu.decode_batch_device(t, fs, fo, fl, W, H, C, C, out=outs[1])
    took = time.perf_counter() - t0
    sleeping = not a.query()
    torch.cuda.synchronize()
    assert sleeping and took < 0.2, f"the call on stream b took {took:.3f} s (stream a still busy: {sleeping})"
    want = np.stack([gpu.fpng_decode_memory(f, C)[1] for f in files]).reshape(N, H, W, C)
    for o, st in zip(outs, (st_a, st_b)):
        assert int(st.abs().sum()) == 0 and np.array_equal(o.cpu().numpy(), want)
