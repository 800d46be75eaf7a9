"""Seeded edge cases of the label-map decode (decode_nearest_kernel, the index store of png_unfilter_ext_kernel<T> and
png_unfilter_kernel<T>): the nearest kernel's grid-stride carry, its fp32 source index past 2^23, its stores into strided
layouts at every row-end residue, 64-bit offsets past 4 GiB, and the index store at band, Adam7 pass and sub-byte edges.

Every case names the construct it exists to reach and reports the numbers that show it does: the launch grid and each thread's
step, the output indices where the fp32 index differs from exact arithmetic, byte offsets past 2^32, band and pass counts.
tests/test_decode_label_edges_cpu.py checks those numbers; tests/test_decode_label_edges_gpu.py compares the kernels with
test_decode_labels_cpu's models (nearest_src, nearest_model, index_model)."""
from __future__ import annotations

import numpy as np

import decode_edges as de
import pngwrite_formats as pf
from test_decode_labels_cpu import nearest_src

NEAREST_THREADS = 256           # decode_nearest_kernel: threads per CTA, each one group of 4 output pixels of a row
GRID_X = 65535                  # the launch caps gridDim.x; each thread then steps by GRID_X * NEAREST_THREADS groups
STEP = GRID_X * NEAREST_THREADS
FOUR_GIB = 1 << 32
MODES = ("nearest", "nearest-exact")


# ---- grid-stride loop ------------------------------------------------------------------------------------------------------------
def nearest_grid(out_h, out_w):
    """decode_nearest_kernel's launch for an out_h x out_w output: groups per row gx, groups, the grid's thread count (the step),
    and the (row, group) step (dy, dq) each thread carries forward"""
    gx = -(-out_w // 4)
    groups = gx * out_h
    step = min(-(-groups // NEAREST_THREADS), GRID_X) * NEAREST_THREADS
    return dict(gx=gx, groups=groups, step=step, dy=step // gx, dq=step % gx)


def carry_steps(out_h, out_w, threads=None):
    """(iterations, carries) per thread of the first `threads` (default all) threads: how often the loop body runs, and how often
    the `xq >= gx` carry fires.  Computed from the same integer rule as the kernel, without the kernel's running sums."""
    g = nearest_grid(out_h, out_w)
    t = np.arange(g["step"] if threads is None else threads, dtype=np.int64)
    iters = np.maximum(0, -(-(g["groups"] - t) // g["step"]))
    xq0 = t % g["gx"]
    # after k steps xq0 + k dq has wrapped floor((xq0 + k dq) / gx) times, once per carry (dq < gx)
    carries = (xq0 + np.maximum(iters - 1, 0) * g["dq"]) // g["gx"]
    return iters, carries


GRID_CASES = (
    ("iterates_twice_with_and_without_carry", (16384, 8195)),
    ("tall_no_carry", (1 << 24, 1)),
    ("carry_on_almost_every_step", (5, 1 << 24)),
)
GRID_SOURCES = ((37, 29, 3, 4), (23, 41, 0, 8), (64, 3, 0, 2))     # (w, h, ctype, depth) of the label files of each call


def grid_boxes(out, k):
    """different boxes for the files of one call, so each blockIdx.y reads another crop"""
    boxes = []
    for j, (w, h, _, _) in enumerate(GRID_SOURCES):
        bh, bw = max(1, h - j - k), max(1, w - 2 * j - k)
        boxes.append((h - bh, (w - bw) // 2, bh, bw))
    return np.array(boxes, np.int32)


# ---- fp32 source index --------------------------------------------------------------------------------------------------------
FP32_OUT = 1 << 24
FP32_LENGTHS = ((1 << 24) - 1, 10_000_019, 5000)


def raw_src(n_in, n_out, exact):
    """the fp32 rule before its clamp: floor(fl(fl(i [+ 0.5]) * fl(n_in / n_out)))"""
    scale = np.float32(n_in) / np.float32(n_out)
    i = np.arange(n_out, dtype=np.float32)
    return np.floor((i + np.float32(0.5) if exact else i) * scale).astype(np.int64)


def exact_src(n_in, n_out, exact):
    """the same index in exact rational arithmetic, clamped: floor((2i + 1) n_in / (2 n_out)) or floor(i n_in / n_out)"""
    i = np.arange(n_out, dtype=np.int64)
    v = (2 * i + 1) * n_in // (2 * n_out) if exact else i * n_in // n_out
    return np.minimum(v, n_in - 1)


def fp32_report(n_in, n_out, exact):
    """(output indices where the fp32 index differs from the exact one, output indices where the clamp to n_in - 1 acts)"""
    fp = nearest_src(n_in, n_out, exact)
    return np.nonzero(fp != exact_src(n_in, n_out, exact))[0], np.nonzero(raw_src(n_in, n_out, exact) > n_in - 1)[0]


def line_pixel(k):
    """the closed-form 8-bit sample at position k of a 1-pixel-wide or 1-pixel-tall source: neighbours always differ, so an index
    off by one changes the value"""
    k = np.asarray(k, np.int64)
    return ((k * 7 + (k >> 8) * 3 + (k >> 16) * 5) & 255).astype(np.uint8)


# ---- output layouts ------------------------------------------------------------------------------------------------------------
LAYOUT_OUT_H = 7
LAYOUT_WIDTHS = (36, 37, 38, 39)            # out_w % 4 = 0, 1, 2, 3: the row end stores 4, 1, 2 and 3 elements
LAYOUTS = ("canvas_odd_offset", "nchw_padded", "hcw")


def layout_variants():
    """(dtype, desired_channels, native, indices) of every output the nearest resize takes: native calls at 1-4 channels into every
    dtype (uint16 source), 8-bit calls at 3 / 4 channels into uint8 and the float types (uint8 source), index calls at 1"""
    out = [(dt, d, True, False) for dt in ("uint8", "uint16", "float16", "bfloat16", "float32") for d in (1, 2, 3, 4)]
    out += [(dt, d, False, False) for dt in ("uint8", "float16", "bfloat16", "float32") for d in (3, 4)]
    out += [(dt, 1, True, True) for dt in ("uint8", "uint16")]
    return out


def layout_strides(layout, n, h, w, d):
    """(size, strides, storage offset, buffer elements) in elements of an [n, h, w, d] view inside a larger guard-filled buffer:
    an NHWC canvas with 3 spare columns and 2 spare rows, entered at an odd element offset; NCHW planes padded by 2 rows and 3
    columns; or HCW rows of w + 1 elements (a permute of an [n, h, d, w + 1] buffer).  Every buffer ends with spare elements."""
    if layout == "canvas_odd_offset":
        pitch = (w + 3) * d
        img = (h + 2) * pitch
        strides, offset = (img, pitch, d, 1), 2 * pitch + 3
    elif layout == "nchw_padded":
        plane = (h + 2) * (w + 3)
        img = d * plane
        strides, offset = (img, w + 3, 1, plane), (w + 3) + 1
    else:
        img = h * d * (w + 1)
        strides, offset = (img, d * (w + 1), 1, w + 1), 0
    return (n, h, w, d), strides, offset, offset + (n + 1) * img


def element_offsets(strides, offset, shape):
    """element offsets of every element of the view: the mask of what a call may write"""
    idx = [np.arange(s, dtype=np.int64) for s in shape]
    grid = np.meshgrid(*idx, indexing="ij")
    return (offset + sum(g * s for g, s in zip(grid, strides))).ravel()


# ---- index store ----------------------------------------------------------------------------------------------------------------
INDEX_FORMATS = [(3, d) for d in (1, 2, 4, 8)] + [(0, d) for d in (1, 2, 4, 8, 16)]
INDEX_WIDTHS = (63, 64, 65)                 # 8k - 1, 8k, 8k + 1
INDEX_HEIGHTS = (31, 32, 33, 63, 65, 97)    # one to four 32-row bands, each side of a band edge
ADAM7_SHAPES = ((9, 271), (40, 280))        # every Adam7 pass two 32-row bands or more


def index_specs():
    """(ctype, depth, interlace, trns, w, h, n_plte, beyond) of the index files: every label format at widths 8k - 1 .. 8k + 1 and
    heights around the band edges; Adam7 files taller than 264 rows; 8-bit gray with a tRNS key (the ext kernel) next to 8-bit
    gray without (png_unfilter_kernel); palettes with fewer entries than the samples reach (beyond: samples past the entry count)"""
    out = []
    for k, (ct, d) in enumerate(INDEX_FORMATS):
        for j, w in enumerate(INDEX_WIDTHS):
            for q, h in enumerate(INDEX_HEIGHTS):
                out.append((ct, d, 0, False, w, h, None, ct == 3 and (j + q) % 3 == 0))
        for w, h in ADAM7_SHAPES:
            out.append((ct, d, 1, False, w, h, None, ct == 3))
    for w in INDEX_WIDTHS:
        for h in (33, 97):
            out.append((0, 8, 0, True, w, h, None, False))
    return out


def index_file(rs, spec, seed):
    """(png, samples [h, w]) of one index spec"""
    ct, d, il, t, w, h, n_plte, beyond = spec
    if beyond:
        top = 1 << d
        n = max(1, top // 3)
        s = rs.randint(0, top, (h, w, 1)).astype(np.uint32)
        s.flat[0] = top - 1                                         # at least one index past the entry count
        plte = rs.randint(0, 256, (n, 3)).astype(np.uint8)
        return pf.make_png(s, 3, d, il, plte=plte, seed=seed), s[..., 0].astype(np.int64)
    png, s, _, _ = pf.case(rs, w, h, ct, d, il, t, seed=seed, n_plte=n_plte)
    return png, s[..., 0].astype(np.int64)


def unfilter_kernel(spec):
    """which kernel unfilters the file: png_unfilter_kernel takes 8-bit gray without tRNS or Adam7, the ext kernel the rest"""
    ct, d, il, t = spec[:4]
    return "png_unfilter_kernel" if (ct, d, il, t) == (0, 8, 0, False) else "png_unfilter_ext_kernel"


def bands(h):
    return -(-h // de.BAND)


# ---- 4 GiB cases ----------------------------------------------------------------------------------------------------------------
BIG_OUT = (37, 29)
BIG_BOXES = (
    ("bottom_right", (de.BIG_H - 48, de.BIG_W - 64, 48, 64)),      # the crop's base row starts 4.4 GB into the intermediate
    ("top_left", (0, 0, 48, 64)),                                  # control
    ("full_height_strip", (0, de.BIG_W - 64, de.BIG_H, 64)),       # base row 0, the source row offsets themselves pass 2^32
)
BIG_PITCH = de.BIG_W * 4 * 2                                       # RGBA uint16 rows of the native intermediate


def big_offsets(box, exact):
    """(byte offset of the crop's first pixel, largest source-row offset from it) in the big file's native RGBA uint16 intermediate"""
    top, left, bh, _ = box
    return (top * de.BIG_W + left) * 8, int(nearest_src(bh, BIG_OUT[0], exact).max()) * BIG_PITCH


BATCH_N, BATCH_OUT = 9, (8192, 8192)        # nearest to RGBA uint16: 512 MiB per file
BATCH_IMAGE = BATCH_OUT[0] * BATCH_OUT[1] * 4 * 2

INDEX_BIG_N, INDEX_BIG_SIDE = 8, 16384      # 8-bit gray id maps decoded to uint16: 512 MiB each
INDEX_BIG_TAIL = ((3, 4, 1, False, 45, 37), (0, 16, 0, False, 33, 19))   # Adam7 4-bit palette, 16-bit gray


def index_big_id(k, y, x):
    """the closed-form id of file k of the index batch at (y, x): blocks of ids that change every row in places, so a misplaced row
    or file shows"""
    y = np.asarray(y, np.int64)
    x = np.asarray(x, np.int64)
    return ((y >> 3) * 7 + (x >> 5) * 13 + k * 29 + ((x ^ y) & 1)) & 255


def index_big_placement():
    """byte offsets of every file of the index batch in the ragged uint16 output: the exclusive scan of align_up(w h 2, 16) in file
    order, as decode_place_kernel computes it"""
    sizes = [INDEX_BIG_SIDE * INDEX_BIG_SIDE * 2] * INDEX_BIG_N + [w * h * 2 for (_, _, _, _, w, h) in INDEX_BIG_TAIL]
    return np.concatenate([[0], np.cumsum([(s + 15) // 16 * 16 for s in sizes])])


def index_big_bytes():
    return int(index_big_placement()[-1])
