"""GPU tests of the batch entry points at the file counts they are sold for, and with calls that overlap.

Every call is checked file by file against the oracle: encoded bytes, sizes and slot offsets, compacted offsets and bytes,
container-walk rows, decoded pixels and statuses, ragged output offsets against placement(), and the guard bytes a call must
not write.  The file counts cross every point where the kernels change how they cover the files: 128 files per CTA of the
container walk and status kernels, 1024 files per round of the one-CTA scans (decode_place_kernel, compact_offsets_kernel),
65535 (the grid.y limit of the per-file grids), and more than three chunks of 65535 files in the pipelined host paths.  The
first pixel of every image holds its index, so a file written to, or decoded from, another file's place changes bytes.  Each
device call must launch as many kernels at every file count as it does for one file.

The first two tests overlap calls: chains on three streams enqueued while the device is still busy, and four host threads with a
stream each.  All device calls share one set of workspaces; overlapping calls must compute what the same calls compute one at a
time.  They come first so that, in file order, a larger call has to grow a workspace that an earlier queued call still uses."""
import ctypes as C
import threading
import traceback

import numpy as np
import pytest

from test_decode_device_gpu import packed_device, to_device
from test_decode_ragged_gpu import GUARD, pack_at, placement
from test_encode_ragged_gpu import launches

pytestmark = pytest.mark.gpu

NOT_FPNG, INVALID_ARG, HEADER_CRC32, SHAPE_MISMATCH, OUT_OF_SPACE, ADLER_MISMATCH = 1, 2, 4, 100, 101, 102
NS = [1, 127, 128, 129, 1023, 1024, 1025, 2049, 65535]
N_MAX = 65535
N_HOST = 3 * 65535 + 1000                 # four chunks of the host batch paths (at most 65535 files per chunk, three slots)
UNIFORM = [(3, 2, 3), (24, 9, 4)]         # (w, h, chans): every file stored / Huffman-coded and stored files mixed
# ragged shapes (w, h, chans, loader): every (chans x loader) class of the ragged encoder, with 13 entries so that shape and
# content kind (index % 4) go through every pairing
RAGGED = [(1, 1, 3, "direct"), (24, 9, 3, "direct"), (16, 3, 3, "staged"), (5, 4, 3, "planar"), (7, 2, 3, "direct"),
          (16, 9, 3, "planar"), (1, 3, 4, "planar"), (24, 9, 4, "staged"), (4, 5, 4, "staged"), (13, 6, 4, "direct"),
          (9, 1, 4, "planar"), (3, 2, 4, "direct"), (12, 9, 4, "staged")]
MAX_W, MAX_H = 24, 9
WIDE = (40, 2, 3)                         # wider than MAX_W: SHAPE_MISMATCH in the ragged decode
# failing files of the decode calls, on both sides of 128 (one CTA of the walk and status kernels) and of 1024 (one round of the
# placement scan): a damaged zlib header ("stream", NOT_FPNG), a valid file of another shape, a size of 0
FAILS = {3: "stream", 127: "shape", 1000: "empty", 1023: "shape", 1024: "stream", 1030: "shape", 1100: "empty", 2048: "stream",
         40000: "shape", 65534: "empty"}


# ---- corpus --------------------------------------------------------------------------------------------------------------
def _mix(x):
    """a 32-bit integer hash, elementwise"""
    x = np.asarray(x, np.uint32)
    x = x ^ (x >> np.uint32(16)); x = x * np.uint32(0x7FEB352D)
    x = x ^ (x >> np.uint32(15)); x = x * np.uint32(0x846CA68B)
    return x ^ (x >> np.uint32(16))


def make_images(idx, w, h, c):
    """images idx of one shape, uint8 [len(idx), h, w, c].  Content by idx % 4: gradient plus noise (g1), runs of one colour two
    rows long, zero, uniform noise (g2, stored blocks).  The first three bytes then hold the index."""
    i = np.asarray(idx, np.uint32).reshape(-1, 1, 1, 1)
    y = np.arange(h, dtype=np.uint32).reshape(1, -1, 1, 1)
    x = np.arange(w, dtype=np.uint32).reshape(1, 1, -1, 1)
    ch = np.arange(c, dtype=np.uint32).reshape(1, 1, 1, -1)
    pos = (y * np.uint32(w) + x) * np.uint32(4) + ch
    g1 = x * np.uint32(29) + y * np.uint32(71) + ch * np.uint32(101) + i * np.uint32(7) + _mix(i * np.uint32(65599) + pos) % np.uint32(7)
    runs = _mix(i * np.uint32(131) + (y >> np.uint32(1)) * np.uint32(8) + ch) + x * np.uint32(0)
    g2 = _mix((i << np.uint32(12)) ^ pos ^ np.uint32(0x9E3779B9))
    kind = i % np.uint32(4)
    px = np.where(kind == 0, g1, np.where(kind == 1, runs, np.where(kind == 2, np.uint32(0), g2)))
    out = np.ascontiguousarray(np.broadcast_to(px, (i.shape[0], h, w, c)).astype(np.uint8))
    flat = out.reshape(i.shape[0], -1)
    for k in range(3):
        flat[:, k] = (i.reshape(-1) >> np.uint32(8 * k)) & np.uint32(255)
    return out


def images_of_shape(idx, w, h, c, step=4096):
    idx = np.asarray(idx)
    return np.concatenate([make_images(idx[a:a + step], w, h, c) for a in range(0, len(idx), step)])


class Corpus:
    """images and the oracle's files of them; file i is flat[starts[i]:starts[i + 1]]"""

    def __init__(self, oracle, images, flags):
        self.images = images
        self.files = [oracle.encode(im, im.shape[1], im.shape[0], im.shape[2], flags) for im in images]
        self.sizes = np.array([len(f) for f in self.files], np.int64)
        self.starts = np.concatenate([[0], np.cumsum(self.sizes)])
        self.flat = np.frombuffer(b"".join(self.files), np.uint8)
        self._decoded = {}

    def decoded(self, oracle, d):
        """the oracle's pixels of every file at d channels (a list; uniform corpora: [n, h, w, d])"""
        if d not in self._decoded:
            px = []
            for f in self.files:
                st, p, *_ = oracle.decode(f, d)
                assert st == 0
                px.append(p)
            if isinstance(self.images, np.ndarray):
                px = np.stack(px).reshape(self.images.shape[:3] + (d,))
            self._decoded[d] = px
        return self._decoded[d]


_CACHE = {}


def uniform(oracle, w, h, c, flags=0):
    key = ("uniform", w, h, c, flags)
    if key not in _CACHE:
        n = N_HOST if (w, h, c, flags) == (*UNIFORM[0], 0) else N_MAX
        _CACHE[key] = Corpus(oracle, images_of_shape(np.arange(n), w, h, c), flags)
    return _CACHE[key]


def entry(i):
    return RAGGED[i % len(RAGGED)]


def ragged_images():
    if "ragged_images" not in _CACHE:
        images = [None] * N_MAX
        for e, (w, h, c, _) in enumerate(RAGGED):
            idx = np.arange(e, N_MAX, len(RAGGED))
            for i, im in zip(idx, images_of_shape(idx, w, h, c)):
                images[i] = im
        _CACHE["ragged_images"] = images
    return _CACHE["ragged_images"]


def ragged(oracle, flags=0):
    key = ("ragged", flags)
    if key not in _CACHE:
        _CACHE[key] = Corpus(oracle, ragged_images(), flags)
    return _CACHE[key]


def ragged_views():
    """device views of the ragged images in one pool: staged images 16-byte aligned, direct ones 3 bytes past a 16-byte
    boundary, planar ones CHW planes seen through permute(1, 2, 0)"""
    import torch
    if "ragged_views" not in _CACHE:
        images = ragged_images()
        offs, at = [], 0
        for i, im in enumerate(images):
            at = (at + 15) // 16 * 16 + (3 if entry(i)[3] == "direct" else 0)
            offs.append(at)
            at += im.size
        pool = np.zeros(at, np.uint8)
        for i, (o, im) in enumerate(zip(offs, images)):
            pool[o:o + im.size] = (im.transpose(2, 0, 1) if entry(i)[3] == "planar" else im).reshape(-1)
        dev = torch.from_numpy(pool).cuda()
        views = []
        for i, (o, im) in enumerate(zip(offs, images)):
            h, w, c = im.shape
            v = dev[o:o + im.size]
            views.append(v.view(c, h, w).permute(1, 2, 0) if entry(i)[3] == "planar" else v.view(h, w, c))
        torch.cuda.synchronize()
        _CACHE["ragged_views"] = views
    return _CACHE["ragged_views"]


def ragged_class(i):
    w, h, c, loader = entry(i)
    return (c, loader)


def slot_offsets(oracle, first, n):
    """encode_ragged_device's slot offsets of ragged images first..first+n-1: the exclusive prefix of max_encoded_size rounded
    up to 16 bytes, the total last"""
    slot = np.array([(oracle.max_encoded_size(w, h, c) + 15) // 16 * 16 for (w, h, c, _) in RAGGED], np.int64)
    return np.concatenate([[0], np.cumsum(slot[np.arange(first, first + n) % len(RAGGED)])])


# ---- checks --------------------------------------------------------------------------------------------------------------
def ranges(starts, lengths):
    """the concatenated index ranges [starts[k], starts[k] + lengths[k])"""
    starts, lengths = np.asarray(starts, np.int64), np.asarray(lengths, np.int64)
    ends = np.cumsum(lengths)
    return np.repeat(starts - (ends - lengths), lengths) + np.arange(int(ends[-1]) if len(ends) else 0)


def same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    diff = (got != want).reshape(len(got), -1).any(1) if got.ndim > 1 else got != want
    bad = np.flatnonzero(diff)
    assert bad.size == 0, f"{what}: {bad.size} of {len(got)} differ, first at {bad[:6].tolist()}: got {got[bad[0]]}, want {want[bad[0]]}"


def check_bytes(buf, want_at, files_flat, sizes, what):
    """file k's sizes[k] bytes at buf[want_at[k]:] equal files_flat's k-th file"""
    got = buf[ranges(want_at, sizes)]
    bad = np.flatnonzero(got != files_flat)
    if bad.size:
        k = int(np.searchsorted(np.cumsum(sizes), bad[0], side="right"))
        raise AssertionError(f"{what}: {bad.size} bytes differ, the first in file {k}")


def idat(gpu, f):
    st, _, _, _, io, il = gpu.get_info_ex(f)
    assert st == 0
    return io, il


def damage_stream(gpu, f):
    """the zlib header byte flipped: NOT_FPNG (and the IDAT CRC no longer matches)"""
    io, _ = idat(gpu, f)
    b = bytearray(f); b[io + 8] ^= 0xFF
    return bytes(b)


def damage_crc(gpu, f):
    """the IDAT CRC flipped: the stream and the pixels are intact"""
    io, il = idat(gpu, f)
    b = bytearray(f); b[io + 8 + il] ^= 1
    return bytes(b)


def damage_adler(gpu, oracle, f):
    """a byte of the zlib Adler-32 flipped and the IDAT CRC recomputed: the pixels are intact"""
    io, il = idat(gpu, f)
    b = bytearray(f); b[io + 8 + il - 2] ^= 0x10
    b[io + 8 + il:io + 12 + il] = oracle.crc32(bytes(b[io + 4:io + 8 + il])).to_bytes(4, "big")
    return bytes(b)


def unwritten(n):
    """a status tensor whose entries the call must all overwrite"""
    import torch
    return torch.full((n,), -7, dtype=torch.int32, device="cuda")


def need_memory(n):
    """a decode call of n files reserves 16 KiB of tables per file (1 GiB at 65535): skip when the device is short of memory"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if n > 32768 and free < 8e9:
        pytest.skip(f"a decode call of {n} files needs about 1 GiB of workspace; {free / 1e9:.1f} GB of device memory free")


def uniform_case(gpu, oracle, shape, d, n, only_stream=False):
    """the first n files of a uniform corpus with FAILS applied; returns (files, statuses, pixels [n, h, w, d] with GUARD where
    the status is not 0)"""
    w, h, c = shape
    U = uniform(oracle, w, h, c)
    other = uniform(oracle, *UNIFORM[1 - UNIFORM.index(shape)])
    files = list(U.files[:n])
    want_st = np.zeros(n, np.int32)
    for i, kind in FAILS.items():
        if i >= n:
            continue
        kind = "stream" if only_stream else kind
        if kind == "stream":
            files[i] = damage_stream(gpu, files[i])
            want_st[i] = oracle.decode(files[i], d)[0]
            assert want_st[i] == NOT_FPNG
        elif kind == "shape":
            files[i], want_st[i] = other.files[i], SHAPE_MISMATCH
        else:
            files[i], want_st[i] = b"", INVALID_ARG
    want_px = U.decoded(oracle, d)[:n].copy()
    want_px[want_st != 0] = GUARD
    return files, want_st, want_px


def ragged_case(gpu, oracle, n):
    """the first n ragged files with FAILS applied ("shape": a file wider than MAX_W); returns (files, oracle statuses and
    pixels of the files at 4 channels, host walk rows)"""
    R = ragged(oracle)
    files = list(R.files[:n])
    px = list(R.decoded(oracle, 4)[:n])
    st = [0] * n
    for i, kind in FAILS.items():
        if i >= n:
            continue
        if kind == "stream":
            files[i] = damage_stream(gpu, files[i])
        elif kind == "shape":
            w, h, c = WIDE
            files[i] = oracle.encode(make_images([i], w, h, c)[0], w, h, c, 0)
        else:
            files[i] = b""
        st[i], px[i] = oracle.decode(files[i], 4)[:2] if files[i] else (INVALID_ARG, None)
    infos = np.array([gpu.get_info_ex(f) if f else (INVALID_ARG, 0, 0, 0, 0, 0) for f in files], np.int64).reshape(n, 6)
    return files, st, px, infos


def check_compact(dst, dst_offsets, cap, flat, sizes, what):
    """a compaction into dst_cap = cap: offsets are the exclusive prefix of the 16-byte aligned sizes, bit 63 of the total is set
    iff a file did not fit, the files that fit are copied, and no other byte of dst changes (but the 16-byte padding of a copied
    file, which comes from its source)"""
    n = len(sizes)
    pad = (sizes + 15) // 16 * 16
    off = np.concatenate([[0], np.cumsum(pad)]).astype(np.uint64)
    got = dst_offsets.cpu().numpy().view(np.uint64)
    same(got[:n], off[:n], what + " offsets")
    total = int(off[n]) | ((1 << 63) if int(off[n]) > cap else 0)
    assert int(got[n]) == total, (what, hex(int(got[n])), hex(total))
    dst = dst.cpu().numpy()
    fit = off[1:] <= cap
    assert fit.all() or not fit[np.argmin(fit):].any(), what            # the files that fit are a prefix
    k = int(fit.sum())
    want = np.full(dst.size, GUARD, np.uint8)
    care = np.ones(dst.size, bool)
    if k:
        want[ranges(off[:k], sizes[:k])] = flat[:int(sizes[:k].sum())]
        care[ranges(off[:k] + sizes[:k].astype(np.uint64), pad[:k] - sizes[:k])] = False
    bad = np.flatnonzero(care & (dst != want))
    assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at {bad[:6].tolist()} (cap {cap}, {k} of {n} files fit)"


def compact_caps(off, n):
    """dst_cap values: the exact total, and a cap that cuts a file of the second round of compact_offsets_kernel (1024 files a
    round) and one of a later round (one of the first round when there is no second)"""
    caps = [int(off[n])]
    if n > 1:
        caps.append(int(off[n // 2]) + 8)
    if n > 1024:
        caps.append(int(off[1024 + (min(n, 2048) - 1024) // 2]) + 8)
    if n > 2048:
        caps.append(int(off[2048 + (n - 2048) // 2]) + 8)
    return caps


# ---- 1. overlapping calls: three streams -----------------------------------------------------------------------------------
class Chain:
    """encode_ragged_device -> compact_packed_device (then a damaged Adler-32 in one file) -> decode_packed_ragged_device ->
    decode_packed_device, over the ragged images first..first+count-1; every output buffer is guard-filled first"""

    def __init__(self, gpu, oracle, first, count, typed, verify):
        import torch
        self.gpu, self.count, self.typed, self.verify = gpu, count, typed, verify
        R = ragged(oracle)
        self.views = ragged_views()[first:first + count]
        self.files = R.files[first:first + count]
        self.sizes_h = R.sizes[first:first + count]
        self.total = int(slot_offsets(oracle, first, count)[-1])
        self.doffs = np.concatenate([[0], np.cumsum((self.sizes_h + 15) // 16 * 16)])
        self.bad = 5                                                     # its Adler-32 is damaged after the compaction
        patch = damage_adler(gpu, oracle, self.files[self.bad])
        self.patch = torch.from_numpy(np.frombuffer(patch, np.uint8).copy()).cuda()
        self.es = 4 if typed else 1
        self.shapes = [im.shape for im in R.images[first:first + count]]
        self.out_bytes = int(sum((h * w * 4 * self.es + 15) // 16 * 16 for (h, w, c) in self.shapes))
        self.mfs = int(self.sizes_h.max())
        self.scale, self.bias = (np.float32([0.5, 1 / 255, 2.0, -1.0]), np.float32([0.25, -0.5, 1.0, 3.0])) if typed else (None, None)

    def steps(self):
        return [self.encode, self.compact, self.decode_ragged, self.decode_packed]

    def encode(self, s):
        import torch
        self.enc = torch.full((self.total,), GUARD, dtype=torch.uint8, device="cuda")
        _, self.offs, self.sizes = self.gpu.encode_ragged_device(self.views, 0, out=self.enc, stream=s)

    def compact(self, s):
        import torch
        self.flat = torch.full((self.total,), GUARD, dtype=torch.uint8, device="cuda")
        _, self.dst_offs = self.gpu.compact_packed_device(self.enc, self.offs, self.sizes, out=self.flat, stream=s)
        o = int(self.doffs[self.bad])
        self.flat[o:o + self.patch.numel()].copy_(self.patch)            # stream-ordered: on the current (chain's) stream

    def decode_ragged(self, s):
        import torch
        self.gpu.set_decode_verify(self.verify[0])
        dt = torch.float32 if self.typed else torch.uint8
        self.rout = torch.full((self.out_bytes // self.es,), -7 if self.typed else GUARD, dtype=dt, device="cuda")
        _, self.roo, self.rinfo, self.rst = self.gpu.decode_packed_ragged_device(
            self.flat, self.dst_offs, self.sizes, 4, out=self.rout, max_file_size=self.mfs, max_w=MAX_W, max_h=MAX_H, stream=s,
            scale=self.scale, bias=self.bias)

    def decode_packed(self, s):
        import torch
        self.gpu.set_decode_verify(self.verify[1])
        w, h, c = UNIFORM[1]
        self.pout = torch.full((self.count, h, w, 4), GUARD, dtype=torch.uint8, device="cuda")
        _, self.pst = self.gpu.decode_packed_device(self.flat, self.dst_offs, self.sizes, w, h, c, 4, max_file_size=self.mfs,
                                                    out=self.pout, stream=s)

    def outputs(self):
        return [self.enc, self.offs, self.sizes, self.flat, self.dst_offs, self.rout, self.roo, self.rinfo, self.rst, self.pout, self.pst]


def check_chain(oracle, ch):
    """a chain's outputs against the oracle"""
    n = ch.count
    enc = ch.enc.cpu().numpy()
    same(ch.sizes.cpu().numpy(), ch.sizes_h, "encoded sizes")
    check_bytes(enc, ch.offs.cpu().numpy()[:n], np.frombuffer(b"".join(ch.files), np.uint8), ch.sizes_h, "encoded files")
    same(ch.dst_offs.cpu().numpy()[:n], ch.doffs[:n], "compacted offsets")
    rst = ch.rst.cpu().numpy()
    want = np.zeros(n, np.int32)
    want[ch.bad] = ADLER_MISMATCH if ch.verify[0] else 0
    same(rst, want, "ragged statuses")
    views = ch.gpu.ragged_views(ch.rout, ch.roo, ch.rinfo, ch.rst, 4)
    for i, v in enumerate(views):
        if want[i] == 0:
            px = oracle.decode(ch.files[i], 4)[1].reshape(v.shape)
            exp = px.astype(np.float32) * ch.scale + ch.bias if ch.typed else px
            assert np.array_equal(v.cpu().numpy(), exp), i
    pst = ch.pst.cpu().numpy()
    want = np.array([0 if (w, h, c) == UNIFORM[1] else SHAPE_MISMATCH for (h, w, c) in ch.shapes], np.int32)
    if want[ch.bad] == 0 and ch.verify[1]:
        want[ch.bad] = ADLER_MISMATCH
    same(pst, want, "packed statuses")


def test_chains_on_three_streams(gpu, oracle):
    """Three chains enqueued step by step round the streams, each step behind a sleep, the verify switch flipped between the
    decode calls.  The second stream's calls need much larger workspaces than the first's just before them, so the
    workspaces are reallocated while the first stream still has work queued.  Every output must equal the same chains run
    one call at a time, and the oracle."""
    import torch
    gpu.set_decode_verify(False)
    # (first image, count, typed ragged decode): 40 files, then 3000, then 400
    chains = [Chain(gpu, oracle, first, count, typed, ((k % 2) == 0, (k % 2) == 1))
              for k, (first, count, typed) in enumerate(((0, 40, False), (100, 3000, False), (3200, 400, True)))]
    streams = [torch.cuda.Stream() for _ in chains]
    torch.cuda.synchronize()
    try:
        for step in range(4):
            for ch, s in zip(chains, streams):
                with torch.cuda.stream(s):
                    torch.cuda._sleep(1 << 28)                           # ~0.1 s of GPU time in front of every step
                    ch.steps()[step](s.cuda_stream)
        torch.cuda.synchronize()
        overlapped = [[t.clone() for t in ch.outputs()] for ch in chains]
        for ch in chains:
            for step in ch.steps():
                step(torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
    finally:
        gpu.set_decode_verify(False)
    for k, (ch, before) in enumerate(zip(chains, overlapped)):
        for j, (a, b) in enumerate(zip(before, ch.outputs())):
            assert torch.equal(a, b), (k, j)
        check_chain(oracle, ch)


# ---- 2. overlapping calls: four host threads ---------------------------------------------------------------------------------
def test_host_threads_with_own_streams(gpu, oracle):
    """Four threads, each with its own stream and its own files, call decode_batch_device (pinned FileDesc staging),
    decode_packed_device and encode_ragged_device for three rounds of different sizes."""
    import torch
    w, h, c = UNIFORM[1]
    U = uniform(oracle, w, h, c)
    R = ragged(oracle)
    px = U.decoded(oracle, 4)
    views = ragged_views()
    counts = (30, 1500, 300)
    plans = [[(t * 12000 + r * 2000, counts[(t + r) % 3]) for r in range(3)] for t in range(4)]
    errors = []

    def worker(t):
        s = torch.cuda.Stream()
        try:
            for r, (a, k) in enumerate(plans[t]):
                files = U.files[a:a + k]
                with torch.cuda.stream(s):
                    tb, _, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, "cuda")
                    px1, st1 = gpu.decode_batch_device(tb, sizes, ofs, lens, w, h, c, 4)
                    data, offsets, dsizes = packed_device(files)
                    px2, st2 = gpu.decode_packed_device(data, offsets, dsizes, w, h, c, 4, max_file_size=int(U.sizes[a:a + k].max()))
                    enc, eoffs, esizes = gpu.encode_ragged_device(views[a:a + k])
                s.synchronize()
                for name, (p, st) in (("decode_batch_device", (px1, st1)), ("decode_packed_device", (px2, st2))):
                    if not (st.cpu().numpy() == 0).all() or not np.array_equal(p.cpu().numpy(), px[a:a + k]):
                        errors.append((t, r, name))
                eo = eoffs.cpu().numpy()
                if not np.array_equal(eo, slot_offsets(oracle, a, k)) or not np.array_equal(esizes.cpu().numpy(), R.sizes[a:a + k]):
                    errors.append((t, r, "encode_ragged_device offsets or sizes"))
                elif not np.array_equal(enc.cpu().numpy()[ranges(eo[:k], R.sizes[a:a + k])], R.flat[R.starts[a]:R.starts[a + k]]):
                    errors.append((t, r, "encode_ragged_device bytes"))
        except Exception:
            errors.append((t, traceback.format_exc()))

    torch.cuda.synchronize()
    ts = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors, errors[:4]


# ---- 3. encode and compaction --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("shape", UNIFORM, ids=lambda s: "%dx%dx%d" % s)
def test_encode_batch_device_and_compact(gpu, oracle, shape, n):
    import torch
    from fpng_b200._lib import lib
    w, h, c = shape
    for flags in (0, 1):
        U = uniform(oracle, w, h, c, flags)
        dev = torch.from_numpy(U.images[:n]).cuda()
        base, _ = launches(gpu, lambda: gpu.encode_batch_device(dev[:1], flags))
        cnt, (out, sizes) = launches(gpu, lambda: gpu.encode_batch_device(dev, flags))
        assert cnt == base, (flags, cnt, base)
        same(sizes.cpu().numpy(), U.sizes[:n], f"sizes, flags {flags}")
        stride = out.stride(0)
        check_bytes(out.cpu().numpy().reshape(-1), np.arange(n) * stride, U.flat[:U.starts[n]], U.sizes[:n], f"files, flags {flags}")
        off = np.concatenate([[0], np.cumsum((U.sizes[:n] + 15) // 16 * 16)])
        for cap in compact_caps(off, n):
            dst = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
            doffs = torch.empty((n + 1,), dtype=torch.int64, device="cuda")
            s = torch.cuda.current_stream().cuda_stream

            def compact(k):
                return lib().fpngb_compact_batch_device(out.data_ptr(), stride, sizes.data_ptr(), k, dst.data_ptr(), cap, doffs.data_ptr(), s)
            base, _ = launches(gpu, lambda: compact(1))
            dst.fill_(GUARD)
            cnt, rc = launches(gpu, lambda: compact(n))
            assert rc == 0 and cnt == base, (rc, cnt, base)
            check_compact(dst, doffs, cap, U.flat, U.sizes[:n], f"compact_batch_device flags {flags} cap {cap}")


@pytest.mark.parametrize("n", NS)
def test_encode_ragged_device_and_compact(gpu, oracle, n):
    import torch
    views = ragged_views()[:n]
    classes = {}
    for i in range(n):
        classes.setdefault(ragged_class(i), i)
    one_per_class = [views[i] for i in sorted(classes.values())]
    want_offs = slot_offsets(oracle, 0, n)
    total = int(want_offs[-1])
    for flags in (0, 1):
        R = ragged(oracle, flags)
        base, _ = launches(gpu, lambda: gpu.encode_ragged_device(one_per_class, flags))
        buf = torch.full((total + 64,), GUARD, dtype=torch.uint8, device="cuda")
        cnt, (_, offsets, sizes) = launches(gpu, lambda: gpu.encode_ragged_device(views, flags, out=buf[:total]))
        assert cnt == base, (flags, cnt, base, len(classes))
        same(offsets.cpu().numpy(), want_offs, f"slot offsets, flags {flags}")
        same(sizes.cpu().numpy(), R.sizes[:n], f"sizes, flags {flags}")
        b = buf.cpu().numpy()
        check_bytes(b, want_offs[:n], R.flat[:R.starts[n]], R.sizes[:n], f"files, flags {flags}")
        assert (b[total:] == GUARD).all(), "a byte past the total was written"
        off = np.concatenate([[0], np.cumsum((R.sizes[:n] + 15) // 16 * 16)])
        for cap in compact_caps(off, n):
            dst = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
            base, _ = launches(gpu, lambda: gpu.compact_packed_device(buf, offsets, sizes[:1], out=dst[:cap]))
            dst.fill_(GUARD)
            cnt, (_, doffs) = launches(gpu, lambda: gpu.compact_packed_device(buf, offsets, sizes, out=dst[:cap]))
            assert cnt == base, (cnt, base)
            check_compact(dst, doffs, cap, R.flat, R.sizes[:n], f"compact_packed_device flags {flags} cap {cap}")


# ---- 4. container walk and decode ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", NS)
def test_get_info_batch_device(gpu, oracle, n):
    files, _, _, infos = ragged_case(gpu, oracle, n)
    data, offsets, sizes = packed_device(files, odd=True)
    base, _ = launches(gpu, lambda: gpu.get_info_batch_device(data, offsets, sizes[:1]))
    cnt, info = launches(gpu, lambda: gpu.get_info_batch_device(data, offsets, sizes))
    assert cnt == base
    same(info.cpu().numpy().view(np.uint32).astype(np.int64), infos, "walk rows")


@pytest.mark.parametrize("n", NS)
def test_decode_batch_device(gpu, oracle, n):
    """the host-walked call: every file goes up in one pinned FileDesc upload"""
    import torch
    need_memory(n)
    w, h, c = UNIFORM[1]
    files, want_st, want_px = uniform_case(gpu, oracle, UNIFORM[1], 4, n, only_stream=True)
    t, _, sizes, ofs, lens, *_ = gpu.pack_files_for_device(files, "cuda")

    def call(k):
        out = torch.full((k, h, w, 4), GUARD, dtype=torch.uint8, device="cuda")
        return out, gpu.decode_batch_device(t[:k], sizes[:k], ofs[:k], lens[:k], w, h, c, 4, out=out, status=unwritten(k))[1]
    base, _ = launches(gpu, lambda: call(1))
    cnt, (out, st) = launches(gpu, lambda: call(n))
    assert cnt == base
    same(st.cpu().numpy(), want_st, "statuses")
    same(out.cpu().numpy(), want_px, "pixels")


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("shape", UNIFORM, ids=lambda s: "%dx%dx%d" % s)
def test_decode_packed_device(gpu, oracle, shape, n):
    import torch
    need_memory(n)
    w, h, c = shape
    files, want_st, want_px = uniform_case(gpu, oracle, shape, 3, n)
    data, offsets, sizes = packed_device(files)
    mfs = max(len(f) for f in files)

    def call(k):
        out = torch.full((k, h, w, 3), GUARD, dtype=torch.uint8, device="cuda")
        return out, gpu.decode_packed_device(data, offsets, sizes[:k], w, h, c, 3, max_file_size=mfs, out=out, status=unwritten(k))[1]
    base, _ = launches(gpu, lambda: call(1))
    cnt, (out, st) = launches(gpu, lambda: call(n))
    assert cnt == base
    same(st.cpu().numpy(), want_st, "statuses")
    same(out.cpu().numpy(), want_px, "pixels")


def ragged_expect(gpu, files, st, px, infos, offs, base_bytes, bounds, cap, oo):
    """statuses, walk rows and output buffer (cap + 64 bytes) a ragged call must return, and the placement offsets"""
    n = len(files)
    pre, want_offs = placement(gpu, files, offs, base_bytes, 4, *bounds, out_cap=cap)
    want_st = np.array([p if p else s for p, s in zip(pre, st)], np.int32)
    want_info = infos.copy()
    want_info[np.array(pre) == INVALID_ARG] = (INVALID_ARG, 0, 0, 0, 0, 0)
    ok = np.flatnonzero(want_st == 0)
    want_out = np.full(cap + 64, GUARD, np.uint8)
    if ok.size:
        want_out[ranges(oo[ok], [px[i].size for i in ok])] = np.concatenate([px[i] for i in ok])
    return want_st, want_info, want_out, want_offs


def check_ragged(got, want, what):
    out, oo, info, st = got
    want_st, want_info, want_out, want_offs = want
    same(oo, want_offs, what + " out_offsets")
    same(st, want_st, what + " statuses")
    same(info.astype(np.int64), want_info, what + " walk rows")
    bad = np.flatnonzero(out != want_out)
    assert bad.size == 0, f"{what}: {bad.size} output bytes differ, first at {bad[:4].tolist()} (file {int(np.searchsorted(oo[:-1], bad[0], side='right')) - 1})"


@pytest.mark.parametrize("n", NS)
def test_decode_packed_ragged_device(gpu, oracle, n):
    """out_cap cuts a file of the placement scan's second round or a later one: that file is the first OUT_OF_SPACE"""
    import torch
    need_memory(n)
    files, st, px, infos = ragged_case(gpu, oracle, n)
    buf, offs = pack_at(files, np.random.RandomState(n), False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    bounds = (max(len(f) for f in files), MAX_W, MAX_H)
    _, full = placement(gpu, files, offs, len(buf), 4, *bounds, out_cap=1 << 62)
    cap = int(full[-1]) if n <= 1024 else int(full[1024 + (n - 1024) // 2]) + 8

    def call(k, cap):
        out = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
        return (out,) + gpu.decode_packed_ragged_device(data, offsets, sizes[:k], 4, out=out[:cap], max_file_size=bounds[0],
                                                        max_w=MAX_W, max_h=MAX_H)[1:]
    base, _ = launches(gpu, lambda: call(1, 4096))
    cnt, got = launches(gpu, lambda: call(n, cap))
    assert cnt == base
    got = [got[0].cpu().numpy(), got[1].cpu().numpy().view(np.uint64), got[2].cpu().numpy().view(np.uint32), got[3].cpu().numpy()]
    check_ragged(got, ragged_expect(gpu, files, st, px, infos, offs, len(buf), bounds, cap, got[1]), f"n {n}")
    oos = np.flatnonzero(got[3] == OUT_OF_SPACE)
    assert (oos.size == 0) == (n <= 1024) and (n <= 1024 or oos[0] >= 1024), oos[:4]


# ---- 5. a float output and the integrity check at the grid limit --------------------------------------------------------------
def verify_damage(gpu, oracle, files, want_st):
    """damage the checksums of four more files (IDAT CRC at 700 and 30001, Adler-32 at 900 and 50002): their pixels and
    statuses are the oracle's with the switch off; returns the statuses with it on (FAILS' stream damage also breaks the CRC)"""
    verified = np.array(want_st, np.int32)
    for i in (700, 30001):
        files[i] = damage_crc(gpu, files[i])
        verified[i] = HEADER_CRC32
    for i in (900, 50002):
        files[i] = damage_adler(gpu, oracle, files[i])
        verified[i] = ADLER_MISMATCH
    for i, kind in FAILS.items():
        if kind == "stream":
            verified[i] = HEADER_CRC32
    return verified


def test_typed_verified_packed_decode_at_grid_limit(gpu, oracle):
    import torch
    n = N_MAX
    need_memory(n)
    w, h, c = UNIFORM[1]
    files, want_st, want_px = uniform_case(gpu, oracle, UNIFORM[1], 4, n)
    verified = verify_damage(gpu, oracle, files, want_st)
    data, offsets, sizes = packed_device(files)
    scale, bias = np.float32([1 / 255, 0.5, -2.0, 3.0]), np.float32([-0.5, 0.25, 7.0, -1.0])

    def call(k):
        out = torch.full((k, h, w, 4), -7.0, dtype=torch.float32, device="cuda")
        return out, gpu.decode_packed_device(data, offsets, sizes[:k], w, h, c, 4, max_file_size=max(len(f) for f in files), out=out,
                                             status=unwritten(k), scale=scale, bias=bias)[1]
    gpu.set_decode_verify(True)
    try:
        base, _ = launches(gpu, lambda: call(1))
        cnt, (out, st) = launches(gpu, lambda: call(n))
    finally:
        gpu.set_decode_verify(False)
    assert cnt == base
    same(st.cpu().numpy(), verified, "statuses")
    out = out.cpu().numpy()
    for a in range(0, n, 8192):                                         # v * scale + bias, two rounded float32 operations
        sl = slice(a, a + 8192)
        want = np.where((verified[sl] == 0)[:, None, None, None], want_px[sl].astype(np.float32) * scale + bias, np.float32(-7.0))
        same(out[sl], want, f"pixels {a}..")


def test_verified_ragged_decode_at_grid_limit(gpu, oracle):
    import torch
    n = N_MAX
    need_memory(n)
    files, st, px, infos = ragged_case(gpu, oracle, n)
    verified = verify_damage(gpu, oracle, files, st)
    buf, offs = pack_at(files, np.random.RandomState(7), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    bounds = (max(len(f) for f in files), MAX_W, MAX_H)
    cap = int(placement(gpu, files, offs, len(buf), 4, *bounds, out_cap=1 << 62)[1][-1])
    out = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    gpu.set_decode_verify(True)
    try:
        _, oo, info, status = gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out[:cap], max_file_size=bounds[0],
                                                              max_w=MAX_W, max_h=MAX_H)
        torch.cuda.synchronize()
    finally:
        gpu.set_decode_verify(False)
    got = [out.cpu().numpy(), oo.cpu().numpy().view(np.uint64), info.cpu().numpy().view(np.uint32), status.cpu().numpy()]
    check_ragged(got, ragged_expect(gpu, files, list(verified), px, infos, offs, len(buf), bounds, cap, got[1]), "verified")


# ---- 6. the pipelined host paths past three chunks -----------------------------------------------------------------------------
def test_host_batch_paths_past_three_chunks(gpu, oracle):
    """N_HOST tiny files: four chunks of at most 65535 files through three slots, in fpngb_encode_batch_host and
    fpngb_decode_batch_host; the decode has damaged files in every chunk and empty ones that shift the chunk boundaries"""
    from fpng_b200._lib import lib
    need_memory(N_MAX)
    w, h, c = UNIFORM[0]
    U = uniform(oracle, w, h, c)
    n = N_HOST
    assert len(U.files) == n
    stride = oracle.max_encoded_size(w, h, c)
    out = np.full((n, stride), GUARD, np.uint8)
    sizes = np.zeros(n, np.uint32)
    imgs = np.ascontiguousarray(U.images)
    rc = lib().fpngb_encode_batch_host(imgs.ctypes.data_as(C.c_void_p), w * h * c, n, w, h, c, 0, out.ctypes.data_as(C.c_void_p), stride,
                                       sizes.ctypes.data_as(C.c_void_p))
    assert rc == 0
    same(sizes.astype(np.int64), U.sizes, "encoded sizes")
    check_bytes(out.reshape(-1), np.arange(n) * stride, U.flat, U.sizes, "encoded files")

    files = list(U.files)
    want_st = np.zeros(n, np.int32)
    for i in (5, 65534, 65535, 131071, 131072, 196605, n - 1):
        files[i] = damage_stream(gpu, files[i])
        want_st[i] = NOT_FPNG
    for i in (70000, 196000):
        files[i] = b""
        want_st[i] = INVALID_ARG
    flat = np.frombuffer(b"".join(files), np.uint8)
    starts = np.concatenate([[0], np.cumsum([len(f) for f in files])])[:-1]
    need = w * h * 3
    px = np.full((n, need), GUARD, np.uint8)
    rc, ww, hh, cc, st = gpu.decode_batch_host(flat.ctypes.data + starts, [len(f) for f in files], 3, px, need)
    assert (rc, ww, hh, cc) == (0, w, h, c)
    same(st, want_st, "decoded statuses")
    ok = want_st == 0
    same(px[ok], U.decoded(oracle, 3).reshape(n, need)[ok], "decoded pixels")
