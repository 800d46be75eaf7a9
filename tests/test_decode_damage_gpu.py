"""GPU tests of the fpng decode on damaged streams (tests/decode_damage.py): every decode entry point gives the reference's status
for every case, and its pixels where the status is 0, with damage at the subsequence, CTA and link-chunk boundaries where the
decode kernels hand a stream from one to the next.  The same large-file set runs with every speculative start wrong (pre-roll 0)
and with the integrity check on.  A disagreement is accepted only when a token trace of the file
(tests/deflatetrace.py) shows one of the documented deviations of INTEGRATION.md section 7; the test prints how many."""
import hashlib
from collections import Counter

import numpy as np
import pytest

import decode_damage as dd
import deflatetrace

pytestmark = pytest.mark.gpu
GUARD = 0x5A
F16_SENTINEL = 0x7E5A                                   # a NaN payload the decode never produces
CRC, NOT_FPNG, ADLER = 4, 1, 102


def digest(px):
    return None if px is None else hashlib.blake2b(np.ascontiguousarray(px).tobytes(), digest_size=16).digest()


@pytest.fixture(scope="module")
def reference(oracle):
    """the reference where oracle/_ref was built, else the oracle (byte-identical decoder)"""
    import refreplay
    return refreplay.reference("Ref") if refreplay._live_available("Ref") else oracle


@pytest.fixture(scope="module")
def damage(oracle, reference):
    """(cases, bases, {(case index, desired): (status, pixel digest)}) with the reference's answers"""
    cases, bases = dd.corpus(oracle)
    want = {}
    for i, c in enumerate(cases):
        for d in (3, 4):
            st, px = reference.decode(c.file, d)[:2]
            want[(i, d)] = (st, digest(px) if st == 0 else None)
    return cases, bases, want


def deviation(f, chans, w):
    """the documented deviation a token trace of file f shows, or None: a scanline that starts with a match, a stored layout other
    than the reference writer's, or a stream whose tokens run past the end of the file (the reference reads past its buffer)"""
    o, n = dd.idat(f)
    try:
        tr = deflatetrace.trace(f[o + 8:])                            # the reference reads on past the IDAT data
    except deflatetrace.DeflateError as e:
        return "read_past_buffer" if "ends inside" in str(e) else None
    rb = w * chans + 1
    if all(b.btype == 0 for b in tr.blocks):
        lens = [b.stored_len for b in tr.blocks]
        raw = sum(lens)
        writer = [65535] * (raw // 65535) + ([raw % 65535] if raw % 65535 else [])
        return "stored_layout" if lens != writer else None
    for b in tr.blocks:
        at = b.out_start
        for t in b.tokens:
            if isinstance(t, tuple):
                if at % rb == 1:
                    return "row_starts_with_match"
                at += t[0]
            else:
                at += 1
    return None


def shape(gpu, f):
    st, w, h, c, *_ = gpu.get_info_ex(f)
    return st, w, h, c


class Tally:
    def __init__(self):
        self.accepted = Counter()

    def check(self, gpu, c, d, st, px, want, what):
        rst, rdig = want
        if st == rst and (st != 0 or digest(px) == rdig):
            return True
        _, w, _, _ = shape(gpu, c.file)
        dev = deviation(c.file, c.chans, w)
        assert dev is not None, (what, c.name, d, st, rst)
        self.accepted[(what, dev)] += 1
        return False


def test_host_entry_points(gpu, damage):
    """fpng_decode_memory at desired 3 and 4, and decode_files, for every case"""
    cases, bases, want = damage
    t = Tally()
    per = Counter()
    for i, c in enumerate(cases):
        for d in (3, 4):
            st, px = gpu.fpng_decode_memory(c.file, d)[:2]
            t.check(gpu, c, d, st, px, want[(i, d)], "fpng_decode_memory")
            per[(c.where or "-", "ok" if want[(i, d)][0] == 0 else "fail")] += 1
    for d in (3, 4):
        res = gpu.decode_files([c.file for c in cases], d)
        for i, (c, r) in enumerate(zip(cases, res)):
            t.check(gpu, c, d, r[0], r[1], want[(i, d)], "decode_files")
    print(f"\n{len(cases)} cases; decodes per boundary and reference outcome:", dict(sorted(per.items())))
    print("accepted deviations:", dict(t.accepted) or 0)


def _group_batches(cases, bases):
    """{base name: [(case index or None for a clean copy, file)]}: each large base file's mutants, with clean copies first, last and
    between every 24 mutants"""
    out = {}
    for name, (png, *_rest) in bases.items():
        items = [(None, png)]
        for i, c in enumerate(cases):
            if c.group == name or (c.group == "stored" and name == "g1_stored_c3"):
                items.append((i, c.file))
                if len(items) % 25 == 0:
                    items.append((None, png))
        items.append((None, png))
        out[name] = items
    return out


def _pack(files, align):
    offs, at = [], 0
    for f in files:
        at = (at + align - 1) // align * align
        offs.append(at)
        at += len(f)
    buf = np.zeros(at + 16, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(f, np.uint8)
    return buf, offs


def test_device_entry_points(gpu, damage):
    """large-file mutants batched with clean copies: decode_batch_device, the ragged call (uint8, float16, any_png) and the resized
    call at identity size; statuses and pixels as the reference's, failed files' output untouched, clean files as a clean-only call"""
    import torch
    cases, bases, want = damage
    t = Tally()
    s16 = np.array([0.5, 2.0, -1.0, 3.0], np.float32)
    b16 = np.array([0.25, -3.0, 7.0, 1.0], np.float32)
    calls = 0
    for name, items in _group_batches(cases, bases).items():
        png, w, h, c, fl = bases[name]
        files = [f for _, f in items]
        ok_walk = [shape(gpu, f) == (0, w, h, c) for f in files]
        n = len(files)
        clean_idx = [k for k, (i, _) in enumerate(items) if i is None]

        want_clean = {d: digest(gpu.fpng_decode_memory(png, d)[1]) for d in (3, 4)}

        def verdict(k, d, st, px, what):
            i = items[k][0]
            if i is None:
                assert st == 0 and digest(px) == want_clean[d], (what, name, k)
                return True
            return t.check(gpu, cases[i], d, st, px, want[(i, d)], what)

        # decode_batch_device: [n, stride] rows, the host walk's IDAT offsets
        idx = [k for k in range(n) if ok_walk[k]]
        stride = (max(len(files[k]) for k in idx) + 16 + 15) // 16 * 16
        rows = np.zeros((len(idx), stride), np.uint8)
        io, il = [], []
        for r, k in enumerate(idx):
            rows[r, :len(files[k])] = np.frombuffer(files[k], np.uint8)
            info = gpu.get_info_ex(files[k])
            io.append(info[4]); il.append(info[5])
        dev = torch.from_numpy(rows).cuda()
        for d in (3, 4):
            out = torch.full((len(idx), h, w, d), GUARD, dtype=torch.uint8, device="cuda")
            _, st = gpu.decode_batch_device(dev, [len(files[k]) for k in idx], io, il, w, h, c, d, out=out)
            st, out = st.cpu().numpy(), out.cpu().numpy()
            calls += 1
            for r, k in enumerate(idx):
                if verdict(k, d, int(st[r]), out[r] if st[r] == 0 else None, "decode_batch_device") and st[r] != 0:
                    assert (out[r] == GUARD).all(), (name, k)
        for align in (16, 4):
            buf, offs = _pack(files, align)
            data = torch.from_numpy(buf).cuda()
            offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
            sizes = torch.tensor([len(f) for f in files], dtype=torch.int32, device="cuda")
            bounds = dict(max_file_size=max(len(f) for f in files), max_w=w, max_h=h)
            for d in (3, 4):
                slot = (w * h * d + 15) // 16 * 16
                u8_st, u8_px = {}, {}
                for kind in ("uint8", "float16", "any_png"):
                    es = 2 if kind == "float16" else 1
                    fill = (torch.full((n * slot + 64,), F16_SENTINEL, dtype=torch.int16, device="cuda").view(torch.float16) if es == 2
                            else torch.full((n * slot + 64,), GUARD, dtype=torch.uint8, device="cuda"))
                    kw = dict(scale=s16[:d].tolist(), bias=b16[:d].tolist()) if es == 2 else {}
                    out, oo, _, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=fill, any_png=kind == "any_png", **bounds, **kw)
                    calls += 1
                    raw = (out.view(torch.int16) if es == 2 else out).cpu().numpy()
                    st, oo = st.cpu().numpy(), oo.cpu().numpy()
                    for k in range(n):
                        o = int(oo[k]) // es
                        px = raw[o:o + w * h * d]
                        if es == 2:                                     # the typed rule: the uint8 call's status, f(its pixels)
                            assert st[k] == u8_st[k], (name, k, d)
                            if st[k] == 0:
                                e = torch.from_numpy(u8_px[k].astype(np.float32).reshape(-1, d) * s16[:d] + b16[:d]).to(torch.float16)
                                assert np.array_equal(px, e.view(torch.int16).numpy().reshape(-1)), (name, k, d)
                            else:
                                assert (px == np.int16(F16_SENTINEL)).all(), (name, k)
                            continue
                        ok = verdict(k, d, int(st[k]), px if st[k] == 0 else None, f"ragged_{kind}")
                        if ok and st[k] != 0:
                            assert (px == GUARD).all(), (name, kind, k)
                        if kind == "uint8":
                            u8_st[k], u8_px[k] = st[k], px.copy()
                    if kind == "uint8":                                 # clean files: the bytes of a clean-only call
                        cbuf, coffs = _pack([png] * len(clean_idx), align)
                        cdata = torch.from_numpy(cbuf).cuda()
                        cout, coo, _, cst = gpu.decode_packed_ragged_device(
                            cdata, torch.tensor(coffs, dtype=torch.int64, device="cuda"),
                            torch.tensor([len(png)] * len(clean_idx), dtype=torch.int32, device="cuda"), d, **bounds)
                        clean_only = cout.cpu().numpy()[int(coo[0].item()):int(coo[0].item()) + w * h * d]
                        for k in clean_idx:
                            o = int(oo[k])
                            assert np.array_equal(raw[o:o + w * h * d], clean_only), (name, k)
                # resized at identity size, uint8
                out = torch.full((n, h, w, d), GUARD, dtype=torch.uint8, device="cuda")
                _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (h, w), d, out=out, pixel_cap=n * slot, **bounds)
                calls += 1
                st, out = st.cpu().numpy(), out.cpu().numpy()
                for k in range(n):
                    if verdict(k, d, int(st[k]), out[k] if st[k] == 0 else None, "resized") and st[k] != 0:
                        assert (out[k] == GUARD).all(), (name, k)
    print(f"\n{calls} device calls; accepted deviations:", dict(t.accepted) or 0)


def test_speculation_and_write_paths(gpu, damage):
    """the large-file, stored and placed cases through the write and stored-block kernels with the scan's pre-roll at 256 and 0
    (every speculative start wrong on a damaged stream)"""
    from fpng_b200._lib import lib
    L = lib()
    cases, bases, want = damage
    sel = [i for i, c in enumerate(cases) if c.group != "small"]
    t = Tally()
    try:
        for pre in (256, 0):
            assert L.fpngb_debug_decode_preroll(pre) == 0
            L.fpngb_debug_decode_repairs(1)
            for d in (3, 4):
                res = gpu.decode_files([cases[i].file for i in sel], d)
                for i, r in zip(sel, res):
                    t.check(gpu, cases[i], d, r[0], r[1], want[(i, d)], f"pre{pre}")
            print(f"pre-roll {pre}: {L.fpngb_debug_decode_repairs(0)} repaired subsequences")
    finally:
        L.fpngb_debug_decode_preroll(dd.PRE_ROLL)
    print(f"{len(sel)} cases x 2 settings; accepted deviations:", dict(t.accepted) or 0)


def test_verify_switch(gpu, damage, reference):
    """with fpngb_set_decode_verify on: a mutant with a stale IDAT CRC gives 4; with its CRC rewritten, the reference's failure, or
    102 exactly when zlib.adler32 of the filtered stream (rebuilt from the reference's pixels) differs from the stored Adler-32"""
    import zlib
    cases, bases, want = damage
    stale = [i for i, c in enumerate(cases) if not c.crc_ok]
    fixed = {}
    for i, c in enumerate(cases):
        o, n = dd.idat(c.file)
        fixed[i] = dd.with_idat(c.file, c.file[o + 8:o + 8 + n])
    outcome = Counter()
    try:
        gpu.set_decode_verify(True)
        for chans in (3, 4):
            idx = [i for i in stale if cases[i].chans == chans]
            res = gpu.decode_files([cases[i].file for i in idx], chans)
            assert all(r[0] == CRC and r[1] is None for r in res)
            outcome["stale_crc"] += len(idx)
            idx = [i for i in range(len(cases)) if cases[i].chans == chans]
            res = gpu.decode_files([fixed[i] for i in idx], chans)
            for i, r in zip(idx, res):
                c = cases[i]
                rst, rpx = reference.decode(fixed[i], chans)[:2]
                if rst != 0:
                    exp = rst
                else:
                    _, w, h, _ = shape(gpu, fixed[i])
                    stored = (fixed[i][dd.idat(fixed[i])[0] + 10] & 6) == 0          # BTYPE of the first block
                    data = dd.filtered_from_pixels(rpx.reshape(h, w, chans), stored)
                    exp = ADLER if zlib.adler32(data) & 0xFFFFFFFF != dd.stored_adler(fixed[i]) else 0
                if r[0] != exp:
                    _, w, *_ = shape(gpu, fixed[i])
                    assert deviation(fixed[i], chans, w) is not None, (c.name, r[0], exp)
                    outcome["accepted_deviation"] += 1
                    continue
                if exp == 0:
                    assert digest(r[1]) == digest(rpx), c.name
                outcome[{0: "ok", ADLER: "adler"}.get(exp, "stream")] += 1
    finally:
        gpu.set_decode_verify(False)
    print("\nverify switch outcomes:", dict(outcome))
    assert outcome["adler"] > 0 and outcome["stale_crc"] > 0
