"""Seeded edge cases of the resized and native decodes (decode_resize_kernel, unfilter_typed_kernel, png_unfilter_kernel<T, true>,
png_unfilter_ext_kernel<T, true>), a sparse float64 model of the resize that computes only the output rows it is asked for, an fp32
emulation of the kernel's summation order, and the error bound E that the GPU comparisons use.

Every case names the construct it exists to reach and reports the numbers that show it does: tiles of the resize grid, tap counts,
the byte offset of the first source row read.  tests/test_decode_edges_cpu.py checks those numbers and the bound; the GPU file
compares the kernels with the model.

The error bound
---------------
The header lets the resize sum "in fp32, in any order".  For one output channel the kernel computes, with raw fp32 weights a_j
(tap_weight) and integer source values p (exact in fp32: at most 65535):

  horizontal, per source row:  h = fl(s_x * norm_x),  s_x = an fmaf chain of nx terms a_j * p_j,
                               norm_x = fl(1 / S_x),  S_x = a recursive fp32 sum of the nx raw weights;
  vertical:                    o = fl(s_y * norm_y),  s_y = an fmaf chain of ny terms b_r * h_r,  norm_y likewise.

With u = 2^-24 and Higham's gamma_k = k u / (1 - k u) (Accuracy and Stability of Numerical Algorithms, 2nd ed., section 3.1):
  * an fmaf chain of n terms rounds once per term, so s_x = sum_j a_j p_j (1 + theta_n^(j)), |theta_n| <= gamma_n;
  * S_x of nonnegative terms is sum_j a_j (1 + theta_(n-1)^(j)), so S_x = S (1 + theta_(n-1)) with S the exact sum; the reciprocal
    and the product add one rounding each.  By Higham's lemma 3.3 ((1 + theta_j) / (1 + theta_k) = 1 + theta_(j+k)):
        h = sum_j (a_j / S) p_j (1 + theta_(2 nx + 1)^(j)),  so |h - h*| <= gamma_(2 nx + 1) * sum_j w_j |p_j| <= gamma_(2 nx + 1) M
    where w_j = a_j / S are the model's normalised weights (nonnegative, summing to 1), h* the exact row value and M = max |p|.
  * the vertical pass applies the same argument to the h_r: o = sum_r v_r h_r (1 + theta_(2 ny + 1)^(r)), hence
        |o - r| <= sum_r v_r (|h_r - h*_r| (1 + gamma_(2 ny + 1)) + |h*_r| gamma_(2 ny + 1))
                <= M (gamma_(2 nx + 1) + gamma_(2 ny + 1) + gamma_(2 nx + 1) gamma_(2 ny + 1)) <= M gamma_(2 (nx + ny) + 2)
    using gamma_a + gamma_b + gamma_a gamma_b <= gamma_(a+b) (Higham, lemma 3.3).
So E = gamma_(2 (nx + ny) + 2) * M: the shape (c1 (nx + ny) + c2) u M with c1 = c2 = 2 (times 1 / (1 - k u), under 1.001 for every
case here).  The model's weights are the kernel's raw fp32 weights normalised in float64, so E covers the whole difference; a span
whose raw weights sum to 0 gives norm 1 in the kernel and 0 in both.  Native calls divide by 257 after this; the comparisons add
that rounding and the storage rounding of the output type on top of E.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

F32 = np.float32
U = 2.0 ** -24
TILE = 32                       # decode_resize_kernel: 32 x 32 output pixels per tile
GRID_X = 65535                  # the launch caps gridDim.x; the tile loop strides by it
UNFILTER_CTA_PX = 512           # unfilter_typed_kernel: 128 threads x 4 pixels
ROWS_AHEAD = 8                  # unfilter_typed_kernel's delta rows per load
BAND = 32                       # png_unfilter_kernel / png_unfilter_ext_kernel: rows per wavefront band


def gamma(k):
    k = np.asarray(k, np.float64)
    return k * U / (1 - k * U)


def bound(nx, ny, m):
    """E: the largest |kernel - float64 model| of an output with nx horizontal and ny vertical taps and sources of at most m"""
    return gamma(2 * (np.asarray(nx) + np.asarray(ny)) + 2) * m


# ---- per-axis spans, as the kernel computes them --------------------------------------------------------------------------------
def spans(inp, out, aa, idx, exact_center=False):
    """(lo int64 [m], size int64 [m], raw fp32 weights [m, k]) of output indices idx along one axis of a crop of length inp.  Each
    operation is one fp32 rounding, as in axis_span / tap_weight; exact_center takes the correctly rounded centre
    fl(scale * (i + 0.5)) instead of fl(scale * fl(i + 0.5)) (they differ for i >= 2^23, where (float)i + 0.5f rounds)."""
    idx = np.asarray(idx, np.int64)
    scale = F32(inp) / F32(out)
    a = bool(aa) and scale >= 1
    sup = scale if a else F32(1)
    inv = F32(1) / scale if a else F32(1)
    if exact_center:
        c = (np.float64(scale) * (idx.astype(np.float64) + 0.5)).astype(F32)
    else:
        c = scale * (idx.astype(F32) + F32(0.5))
    lo = np.maximum((c - sup + F32(0.5)).astype(np.int64), 0)                  # astype truncates toward 0, as (int) does
    hi = np.minimum((c + sup + F32(0.5)).astype(np.int64), inp)
    size = hi - lo
    k = max(int(size.max()), 1)
    j = np.arange(k)
    t = ((j[None, :] + lo[:, None]).astype(F32) - c[:, None] + F32(0.5)) * inv
    w = np.maximum(F32(0), F32(1) - np.abs(t))
    w[j[None, :] >= size[:, None]] = 0
    return lo, size, w


def normalised(w):
    w = w.astype(np.float64)
    s = w.sum(1, keepdims=True)
    return np.where(s != 0, w / np.where(s != 0, s, 1), w)


# ---- the float64 model, row by row -----------------------------------------------------------------------------------------------
def model_rows(fetch, bh, bw, out_h, out_w, aa, rows, cols=None):
    """float64 [len(rows), len(cols), C] resampled values of output rows `rows` (and columns `cols`, default all) of a crop of
    bh x bw source pixels; fetch(r0, r1, c0, c1) returns the crop's rows r0..r1-1, columns c0..c1-1 as [r1-r0, c1-c0, C].  The
    same values as test_decode_resized_cpu.resize_model, without its dense [out, in] matrices."""
    cols = np.arange(out_w) if cols is None else np.asarray(cols, np.int64)
    ylo, ysz, yw = spans(bh, out_h, aa, rows)
    xlo, xsz, xw = spans(bw, out_w, aa, cols)
    yw, xw = normalised(yw), normalised(xw)
    c0 = int(xlo.min())
    c1 = int((xlo + xsz).max())
    out = []
    for q in range(len(rows)):
        src = fetch(int(ylo[q]), int(ylo[q] + max(ysz[q], 1)), c0, c1).astype(np.float64)
        col = np.einsum("r,rwc->wc", yw[q, :src.shape[0]], src)                    # vertical first: the model is separable
        acc = np.zeros((len(cols), col.shape[1]))
        for j in range(xw.shape[1]):
            ok = j < xsz
            acc[ok] += xw[ok, j, None] * col[np.minimum(xlo[ok] + j - c0, col.shape[0] - 1)]
        out.append(acc)
    return np.stack(out)


def emulate_rows(fetch, bh, bw, out_h, out_w, aa, rows, cols=None):
    """the kernel's fp32 order for the same outputs: per source row an fmaf chain of the raw weights (each fmaf one rounding:
    the exact float64 a * b + c rounded once to fp32), times norm_x; then a vertical fmaf chain, times norm_y"""
    cols = np.arange(out_w) if cols is None else np.asarray(cols, np.int64)
    ylo, ysz, yw = spans(bh, out_h, aa, rows)
    xlo, xsz, xw = spans(bw, out_w, aa, cols)
    def norm(w, n):
        s = np.zeros(w.shape[0], F32)
        for j in range(w.shape[1]):
            s = np.where(j < n, (s + w[:, j]).astype(F32), s)
        return np.where(s != 0, F32(1) / np.where(s != 0, s, F32(1)), F32(1)).astype(F32)
    nx, ny = norm(xw, xsz), norm(yw, ysz)
    c0, c1 = int(xlo.min()), int((xlo + xsz).max())
    out = []
    for q in range(len(rows)):
        src = fetch(int(ylo[q]), int(ylo[q] + ysz[q]), c0, c1).astype(np.float64)
        h = np.zeros((src.shape[0], len(cols), src.shape[2]), F32)
        for j in range(xw.shape[1]):
            ok = j < xsz
            v = src[:, np.minimum(xlo + j - c0, src.shape[1] - 1)]
            h = np.where(ok[None, :, None], (xw[None, :, j, None].astype(np.float64) * v + h).astype(F32), h)
        h = (h * nx[None, :, None]).astype(F32)
        acc = np.zeros((len(cols), src.shape[2]), F32)
        for r in range(src.shape[0]):
            acc = (np.float64(yw[q, r]) * h[r].astype(np.float64) + acc).astype(F32)
        out.append((acc * ny[q]).astype(F32))
    return np.stack(out).astype(np.float64)


def array_fetch(px, box=None):
    top, left = (0, 0) if box is None else (int(box[0]), int(box[1]))
    return lambda r0, r1, c0, c1: px[top + r0:top + r1, left + c0:left + c1]


def taps(bh, bw, out_h, out_w, aa, rows, cols=None):
    """(nx [len(cols)], ny [len(rows)]): the span sizes the bound counts"""
    cols = np.arange(out_w) if cols is None else cols
    return spans(bw, out_w, aa, cols)[1], spans(bh, out_h, aa, rows)[1]


def tiles(out_h, out_w):
    return -(-out_w // TILE) * -(-out_h // TILE)


def sample_rows(out_h, n, seed):
    """a seeded sample of output rows: the first, the last and n others"""
    rs = np.random.RandomState(seed)
    return np.unique(np.concatenate([[0, out_h - 1], rs.randint(0, out_h, n)]))


def center_rounds(n_in, n_out, aa, lo=1 << 23, hi=None):
    """output indices in lo..hi whose spans or weights computed with the fp32 centre differ from the float64-exact centre's"""
    idx = np.arange(lo, hi or n_out)
    a, sa, wa = spans(n_in, n_out, aa, idx)
    b, sb, wb = spans(n_in, n_out, aa, idx, exact_center=True)
    k = min(wa.shape[1], wb.shape[1])
    diff = (a != b) | (sa != sb) | (wa[:, :k] != wb[:, :k]).any(1)
    return idx[diff]


# ---- sources ---------------------------------------------------------------------------------------------------------------------
def smooth(h, w, c, seed, depth=8):
    """a compressible [h, w, c] image with detail at every scale: a diagonal ramp, a checker of period 3 / 5 and seeded noise"""
    rs = np.random.RandomState(seed)
    y = np.arange(h, dtype=np.int64)[:, None, None]
    x = np.arange(w, dtype=np.int64)[None, :, None]
    ch = np.arange(c, dtype=np.int64)[None, None, :]
    top = (1 << depth) - 1
    v = (x * 7 + y * 3 + ch * 61) % (top + 1) ^ (((x // 3 + y // 5) & 1) * (top // 4)) + rs.randint(0, 4, (h, w, c))
    return np.clip(v, 0, top).astype(np.uint32)


def big_pixel(y, x, c):
    """the closed-form pixel of the 24000 x 23000 RGB file: uint8 of (x, y, c), computable for any crop"""
    y = np.asarray(y, np.int64)
    x = np.asarray(x, np.int64)
    c = np.asarray(c, np.int64)
    return ((x * 3 + y * 7 + c * 85 + ((x ^ y) >> 4) * 29) & 255).astype(np.uint8)


BIG_W, BIG_H = 24000, 23000


def big_fetch(box, chans=4):
    """fetch for a crop of the big file decoded natively: 16-bit domain values, alpha 65535 at 4 channels"""
    top, left = int(box[0]), int(box[1])

    def f(r0, r1, c0, c1):
        y = np.arange(top + r0, top + r1)[:, None, None]
        x = np.arange(left + c0, left + c1)[None, :, None]
        v = big_pixel(y, x, np.arange(3)[None, None, :]).astype(np.int64) * 257
        if chans == 4:
            v = np.concatenate([v, np.full(v.shape[:2] + (1,), 65535, np.int64)], -1)
        return v
    return f


# ---- resize cases ----------------------------------------------------------------------------------------------------------------
@dataclass
class ResizeCase:
    name: str                    # the construct the case reaches
    src: tuple                   # (h, w) of the source image
    out: tuple                   # (out_h, out_w)
    box: tuple = None            # (top, left, height, width), None: the whole image
    aa: bool = True
    native: bool = False
    chans: int = 3               # channels of the resize (DST)
    rows: np.ndarray = field(default=None, repr=False)  # output rows compared (None: all)

    @property
    def crop(self):
        return self.box or (0, 0) + tuple(self.src)

    def tiles(self):
        return tiles(*self.out)

    def taps(self):
        _, _, bh, bw = self.crop
        rows = np.arange(self.out[0]) if self.rows is None else self.rows
        cols = np.arange(min(self.out[1], 4096))
        nx, ny = taps(bh, bw, self.out[0], self.out[1], self.aa, rows, cols)
        return int(nx.max()), int(ny.max())

    def first_row_offset(self):
        """byte offset, from the file's base in the ragged intermediate, of the first source row the kernel reads for the rows compared"""
        top, _, bh, _ = self.crop
        rows = np.arange(self.out[0]) if self.rows is None else self.rows
        lo = spans(bh, self.out[0], self.aa, rows)[0]
        return (top + int(lo.max())) * self.src[1] * self.chans * (2 if self.native else 1)


def tile_loop_cases():
    """outputs with more tiles than the grid holds; 2^24 x 1 also reaches output indices >= 2^23"""
    out = []
    for h in (3, 5000):
        out.append(ResizeCase(f"tile_loop_2^24x1_from_h{h}", (h, 5 if h > 3 else 37), (1, 1 << 24)))
    out.append(ResizeCase("tile_loop_8224x8192", (48, 64), (8192, 8224), rows=sample_rows(8192, 14, 3)))
    return out


def tap_cases():
    """tap counts in the thousands, whole and as a crop, antialias on and off"""
    out = []
    for (h, w), size in (((8, 3840), (1, 1)), ((8, 3840), (2, 3)), ((2160, 8), (1, 1)), ((2, 16384), (1, 1)), ((1080, 1920), (5, 7))):
        for aa in (True, False):
            out.append(ResizeCase(f"taps_{w}x{h}_to_{size[1]}x{size[0]}_aa{int(aa)}", (h, w), size, aa=aa))
            box = (h // 4, w // 8, h - h // 4 - (h > 2), w - w // 8 - 3)                 # a crop ending short of the last row / column
            out.append(ResizeCase(f"taps_{w}x{h}_crop_to_{size[1]}x{size[0]}_aa{int(aa)}", (h, w), size, box=box, aa=aa))
    return out


def native_tap_cases():
    out = []
    for (h, w, c), size in (((16, 4096, 1), (1, 1)), ((1024, 1024, 4), (3, 3))):
        for aa in (True, False):
            out.append(ResizeCase(f"native_taps_{w}x{h}x{c}_aa{int(aa)}", (h, w), size, aa=aa, native=True, chans=c))
            out.append(ResizeCase(f"native_taps_{w}x{h}x{c}_crop_aa{int(aa)}", (h, w), size, box=(h // 2, 1, h - h // 2, w - 2), aa=aa,
                                  native=True, chans=c))
    return out


def crop_boxes(h, w):
    """1 x 1 boxes at each corner (the last at (h-1, w-1)), boxes whose last tap row is the image's last row, and the full image
    minus one row and one column"""
    return [(0, 0, 1, 1), (0, w - 1, 1, 1), (h - 1, 0, 1, 1), (h - 1, w - 1, 1, 1),
            (h - 7, w - 300, 7, 300), (h - 100, 17, 100, 33), (h - 2, w - 2, 2, 2),
            (1, 1, h - 1, w - 1), (0, 0, h - 1, w - 1)]


CROP_SIZES = ((3, 5), (67, 45))          # up from the small boxes, down from the large ones


def crop_cases(h, w, native=False, chans=3):
    return [ResizeCase(f"crop_{b}_to_{s[1]}x{s[0]}_aa{int(aa)}", (h, w), s, box=b, aa=aa, native=native, chans=chans)
            for s in CROP_SIZES for aa in (True, False) for b in crop_boxes(h, w)]


BIG_BOXES = ((BIG_H - 48, BIG_W - 64, 48, 64), (0, 0, 48, 64))      # rows past 4 GiB of the uint16 intermediate, and a control
BIG_OUT = (37, 29)


def big_cases():
    return [ResizeCase(f"big_intermediate_box_{b[:2]}", (BIG_H, BIG_W), BIG_OUT, box=b, native=True, chans=4) for b in BIG_BOXES]


BATCH_N, BATCH_OUT = 9, (8192, 8192)     # 9 x 512 MiB of RGBA uint16


def batch_bytes():
    return BATCH_N * BATCH_OUT[0] * BATCH_OUT[1] * 4 * 2


# ---- native ragged decode cases --------------------------------------------------------------------------------------------------
FPNG_WIDTHS = (511, 512, 513, 1025, 2047, 2049)
FPNG_HEIGHTS = tuple(range(1, 10)) + (15, 16, 17)


def fpng_shapes():
    """(w, h, c, stored) of the fpng files: widths around one and several unfilter CTAs, heights around the 8 rows loaded ahead"""
    out = []
    for k, w in enumerate(FPNG_WIDTHS):
        for j, h in enumerate(FPNG_HEIGHTS):
            out.append((w, h, 3 + (k + j) % 2, (k + j) % 3 == 0))
    return out


def fpng_image(w, h, c, stored, seed):
    """uint8 [h, w, c]: seeded noise (fpng writes it as stored blocks) or imagegen's gradient with noise (Huffman coded)"""
    import imagegen
    if stored:
        return np.random.RandomState(seed).randint(0, 256, (h, w, c)).astype(np.uint8)
    return imagegen.gradient_noise(w, h, c, seed)


GEN_HEIGHTS = (31, 32, 33, 63, 65, 97)
GEN_WIDTHS = (1, 2, 33, 257)


def general_shapes():
    """(w, h, ctype) of the 8-bit general files of one call: every color type at every shape, so D and the placement vary"""
    return [(w, h, ctype) for h in GEN_HEIGHTS for w in GEN_WIDTHS for ctype in (0, 2, 4, 6)]


def ext_specs():
    """(ctype, depth, interlace, trns, w, h) of the ext files: Adam7 taller than 264 rows (every pass two bands or more), palette
    and gray 1/2/4-bit at widths 8k - 1, 8k, 8k + 1 over several bands, 16-bit files with a color key"""
    out = [(ct, d, 1, False, w, 271) for (ct, d) in ((2, 8), (0, 4), (6, 16), (3, 2)) for w in (9, 40)]
    for ct in (3, 0):
        for d in (1, 2, 4):
            for w in (63, 64, 65):
                out.append((ct, d, 0, ct == 3, w, 70))
    out += [(0, 16, 0, True, 37, 97), (2, 16, 0, True, 33, 65), (2, 16, 1, True, 17, 280)]
    return out


def ext_passes_min_rows(w, h):
    """the fewest rows of any Adam7 pass of a w x h image"""
    import pngwrite_formats as pf
    return min(ph for (_, _, _, _, _, ph) in pf.passes(w, h, 1))
