"""Seeded edge cases of the colour-type reduction (encode_png_device(reduce=True), FPNGB_ENCODE_REDUCE; DESIGN §4.6 "Colour-type
reduction") and a pure-Python model of how reduce_analyze_kernel (csrc/reduce_kernels.cu) cuts an image into pieces, so that every
case can show the construct it reaches:

  * the analysis: CTA b of an image reads pixels [b P, (b + 1) P) in row-major order (P = kRedThreads * kRedIters), thread t at
    step s pixel b P + s kRedThreads + t.  A CTA stops reading once every bit of the `need` mask of the image's (channels, depth)
    class is set in the image's flags.  Colours go to a kReduceSlots-slot shared set, merged into the image's global set at the
    CTA's end; the colour 0x00000000 is a flag bit that counts towards K.
  * the conversion: one thread per 32-bit output word, kRedConvThreads words per CTA over the rows of every changed image.

Most cases are pairs: a base image and the same image with one deciding pixel changed, each with the format reduce_model.choose
gives it.  Nothing here asks the library what the answer is.  tests/test_encode_reduce_edges_cpu.py checks that every case means
what it says; tests/test_encode_reduce_edges_gpu.py runs them through the reduce call.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field

import numpy as np

from reduce_model import choose

# the kernels' partition constants: KERNEL_CONSTANTS ties each to its definition in the sources (checked by the CPU test)
RED_THREADS = 256                # reduce_kernels.cu: threads per analysis CTA, consecutive pixels of one step
RED_ITERS = 32                   # reduce_kernels.cu: steps per analysis CTA
RED_PIXELS = RED_THREADS * RED_ITERS
CONV_THREADS = 256               # reduce_kernels.cu: output words per conversion CTA
SLOTS = 512                      # kernels.cuh: slots of the shared and the global colour set
KERNEL_CONSTANTS = {
    "kRedThreads": ("reduce_kernels.cu", RED_THREADS),
    "kRedIters": ("reduce_kernels.cu", RED_ITERS),
    "kRedConvThreads": ("reduce_kernels.cu", CONV_THREADS),
    "kReduceSlots": ("kernels.cuh", SLOTS),
}
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fpng_b200", "csrc")

# the analysis flags (kernels.cuh)
NOT_REP8, NOT_OPAQUE, NOT_GRAY, OVERFLOW = 1, 2, 4, 64
CLASSES = [(c, d) for c in (1, 2, 3, 4) for d in (8, 16)]
WIDTHS = (1, 3, 255, 256, 257, 8191, 8192, 8193)
CTYPE = {"gray": 0, "palette": 3, "ga": 4, "rgb": 2, "rgba": 6}


def source_constants():
    """{name: value} of KERNEL_CONSTANTS as the sources define them, also inside a multi-declaration
    (`constexpr uint32_t a = 1, b = 2;`)"""
    out = {}
    for name, (fname, _) in KERNEL_CONSTANTS.items():
        with open(os.path.join(CSRC, fname)) as fh:
            m = re.findall(r"constexpr\s+uint32_t\s+(?:[^;]*?,\s*)?\b" + name + r"\s*=\s*(\d+)u?\s*[,;]", fh.read())
        out[name] = int(m[0]) if len(m) == 1 else None
    return out


# ---- the partition ---------------------------------------------------------------------------------------------------------------
def place(p):
    """(CTA, step, thread) of the analysis that reads row-major pixel p of its image"""
    cta, r = divmod(int(p), RED_PIXELS)
    step, thread = divmod(r, RED_THREADS)
    return cta, step, thread


def pixel_at(cta, step, thread):
    return cta * RED_PIXELS + step * RED_THREADS + thread


def analyze_ctas(w, h):
    return -(-w * h // RED_PIXELS)


def conv_words(w, fmt, bits, depth):
    """32-bit words of one reduced row, as reduce_images_locked sizes them"""
    if fmt == "palette" or (fmt == "gray" and depth < 8):
        return -(-w * depth // 32)
    return -(-w * (bits // 8) // 4)


# ---- the early stop --------------------------------------------------------------------------------------------------------------
def need_mask(chans, depth):
    """the evidence reduce_analyze_image waits for before it stops reading: all of it can still change the format"""
    return OVERFLOW | NOT_GRAY | (0 if chans & 1 else NOT_OPAQUE) | (NOT_REP8 if depth == 16 else 0)


def settable(chans, depth):
    """the bits of need_mask an image of the class can set at all (1 channel 8-bit holds at most 256 colours; so does a 1-channel
    16-bit image's key, its high byte)"""
    bits = NOT_GRAY if chans >= 3 else 0
    bits |= NOT_OPAQUE if chans in (2, 4) else 0
    bits |= NOT_REP8 if depth == 16 else 0
    bits |= OVERFLOW if chans >= 2 else 0
    return bits


def can_stop(chans, depth):
    n = need_mask(chans, depth)
    return settable(chans, depth) & n == n


NEVER_STOPS = [(c, d) for (c, d) in CLASSES if c <= 2]      # not-gray is in need and cannot be set: every CTA reads every step
FINAL_WHEN_STOPPED = [(3, 8)]                                  # overflow + not gray leave only RGB8: no late evidence matters


# ---- pixels --------------------------------------------------------------------------------------------------------------------
def as_class(rgba8, chans, depth):
    """uint8 RGBA colours [..., 4] as samples of a (chans, depth) image (8-bit values v as v * 257 at 16 bits)"""
    a = np.asarray(rgba8, np.uint32)
    s = a[..., {1: [0], 2: [0, 3], 3: [0, 1, 2], 4: [0, 1, 2, 3]}[chans]]
    return (s * 257).astype(np.uint16) if depth == 16 else s.astype(np.uint8)


def distinct_rgb(n, seed, gray=False):
    """n distinct opaque colours [n, 4] uint8, none gray-valued (or all gray when gray: n <= 256)"""
    rng = np.random.default_rng(seed)
    if gray:
        g = rng.permutation(256)[:n]
        return np.stack([g, g, g, np.full(n, 255)], 1).astype(np.uint8)
    keys = rng.choice(1 << 24, 2 * n + 16, replace=False)
    c = np.stack([keys >> 16, (keys >> 8) & 255, keys & 255], 1)
    c = c[~((c[:, 0] == c[:, 1]) & (c[:, 1] == c[:, 2]))][:n]
    return np.concatenate([c, np.full((n, 1), 255)], 1).astype(np.uint8)


def colliding_rgb(n, slot=None):
    """n opaque RGB colours [n, 4] whose keys RGB << 8 | 0xFF all hash to one slot of the colour sets, and that slot"""
    rgb = np.arange(1 << 20, dtype=np.uint64) * 13 + 7
    slots = (((rgb << 8 | 0xFF) * 0x9E3779B1) & 0xFFFFFFFF) >> 23
    slot = int(slots[0]) if slot is None else slot
    k = rgb[slots == slot][:n].astype(np.int64)
    assert len(k) == n
    return np.stack([k >> 16, (k >> 8) & 255, k & 255, np.full(n, 255)], 1).astype(np.uint8), slot


def key_of(rgba8):
    c = np.asarray(rgba8, np.uint64)
    return (c[..., 0] << 24 | c[..., 1] << 16 | c[..., 2] << 8 | c[..., 3]).astype(np.uint32)


def fmt_of(img):
    f, bits, depth = choose(img)
    return (f, depth)


# ---- case 1: the deciding pixel at the partition's edges -------------------------------------------------------------------------
MIN_PIXELS = 2 * RED_PIXELS + 1100                 # three CTAs at least, the last one partial unless 8192 divides w * h
FILL_AT = 300                                      # the base colours sit at pixels [300, 300 + n): past step 0, before 7936


def edge_shape(w):
    return -(-MIN_PIXELS // w), w


def edge_positions(h, w):
    """{name: pixel}: the places case 1 puts its deciding pixel"""
    n, ctas = w * h, analyze_ctas(w, h)
    mid = (ctas - 1) // 2
    return {"first": 0, "step0_last_thread": RED_THREADS - 1, "cta0_last_step": pixel_at(0, RED_ITERS - 1, 0),
            "cta0_last": RED_PIXELS - 1, "cta1_first": RED_PIXELS, "mid_cta_last_step": pixel_at(mid, RED_ITERS - 1, 97),
            "last_cta_first": (ctas - 1) * RED_PIXELS, "last": n - 1}


@dataclass
class Case:
    name: str
    base: np.ndarray
    changed: np.ndarray
    pixel: int
    want: tuple                      # (format, depth) of base and of changed, from reduce_model.choose
    want_changed: tuple
    chans: int
    depth: int
    meta: dict = field(default_factory=dict)

    @property
    def place(self):
        return place(self.pixel)


def _image(h, w, chans, depth, background, fills=()):
    """an image of one background colour (8-bit RGBA, or the class's samples given in its dtype), with the colours of
    each (start, colours) of fills written at consecutive pixels from start"""
    bg = np.asarray(background)
    img = np.empty((h * w, chans), np.uint16 if depth == 16 else np.uint8)
    img[:] = bg if bg.shape == (chans,) and bg.dtype == img.dtype else as_class(bg, chans, depth)
    for start, cols in fills:
        cols = np.asarray(cols)
        img[start:start + len(cols)] = cols if cols.shape[-1] == chans and cols.dtype == img.dtype else as_class(cols, chans, depth)
    return img.reshape(h, w, chans)


def _set(img, p, **chan_values):
    """a copy of img with samples of pixel p replaced: r, g, b, a (a is channel chans - 1 of a 2-channel image)"""
    out = img.copy()
    flat = out.reshape(-1, img.shape[2])
    idx = {"r": 0, "g": 1, "b": 2, "a": img.shape[2] - 1}
    for k, v in chan_values.items():
        flat[p, idx[k]] = v
    return out


def _put(img, p, rgba8):
    """a copy of img with pixel p set to an 8-bit RGBA colour (as the class holds it)"""
    out = img.copy()
    out.reshape(-1, img.shape[2])[p] = as_class(rgba8, img.shape[2], 16 if img.dtype == np.uint16 else 8)
    return out


REP8_BREAKERS = (257 * 100 + 1, 257 * 100 - 1, 0x00FF, 0xFF00)


def _edge_variants():
    """[(property, variant, chans, depth, base builder (h, w) -> image, change (image, p, k) -> image)]; k: the position's index"""
    out = []
    all_gray = distinct_rgb(256, 1, gray=True)
    many = distinct_rgb(300, 2)
    ga_pairs = np.stack([np.arange(300) % 256] * 3 + [100 + np.arange(300) // 256], 1).astype(np.uint8)
    # not opaque: alpha 254 (65534) at the pixel
    for c, d in ((2, 8), (2, 16), (4, 8), (4, 16)):
        if d == 8:
            bg, fills = ((100, 100, 100, 255), [(FILL_AT, all_gray)]) if c == 2 else ((10, 20, 30, 255), [(FILL_AT, many)])
        else:
            bg, fills = (np.array([1000, 65535] if c == 2 else [1000, 2000, 3000, 65535], np.uint16), [])
        out.append(("not_opaque", "alpha", c, d, lambda h, w, c=c, d=d, bg=bg, f=fills: _image(h, w, c, d, bg, f),
                    lambda im, p, k, d=d: _set(im, p, a=254 if d == 8 else 65534)))
    # not gray: one of R, G, B moved off the other two
    for c, d in ((3, 8), (3, 16), (4, 8), (4, 16)):
        bg = (100, 100, 100, 255) if d == 8 else np.array([1000] * 3 + [65535] * (c - 3), np.uint16)
        fills = [(FILL_AT, all_gray)] if d == 8 else []
        for ch in "rgb":
            out.append(("not_gray", ch, c, d, lambda h, w, c=c, d=d, bg=bg, f=fills: _image(h, w, c, d, bg, f),
                        lambda im, p, k, ch=ch, d=d: _set(im, p, **{ch: 101 if d == 8 else 1001})))
    # not 8-bit representable in one channel: 257k + 1, 257k - 1, 0x00FF, 0xFF00 (one value per position, in turn)
    for c in (1, 2, 3, 4):
        if c == 1:
            bg, fills = (100, 100, 100, 255), [(FILL_AT, all_gray)]
        elif c == 2:
            bg, fills = (100, 100, 100, 128), [(FILL_AT, ga_pairs)]
        else:
            cols = many.copy()
            cols[:, 3] = 128 if c == 4 else 255
            bg, fills = (10, 20, 30, 128 if c == 4 else 255), [(FILL_AT, cols)]
        for ch in {1: "r", 2: "ra", 3: "rgb", 4: "rgba"}[c]:
            out.append(("not_rep8", ch, c, 16, lambda h, w, c=c, bg=bg, f=fills: _image(h, w, c, 16, bg, f),
                        lambda im, p, k, ch=ch: _set(im, p, **{ch: REP8_BREAKERS[k % len(REP8_BREAKERS)]})))
    # off the lattice: 0/255 + 85 -> 2-bit, {0, 85, 170, 255} + 17 -> 4-bit, 0/255 + 1 -> palette, the 16 4-bit levels + 1 -> gray8
    lat = {"85": ([0, 255], 85), "17": ([0, 85, 170, 255], 17), "1_palette": ([0, 255], 1), "1_gray8": (list(range(0, 256, 17)), 1)}
    for name, (levels, v) in lat.items():
        cols = np.array([[g, g, g, 255] for g in levels], np.uint8)
        for c, d in CLASSES:
            out.append(("lattice", name, c, d, lambda h, w, c=c, d=d, cols=cols: _image(h, w, c, d, (0, 0, 0, 255), [(FILL_AT, cols)]),
                        lambda im, p, k, v=v: _put(im, p, (v, v, v, 255))))
    # the 257th colour: 256 colours (background included), then one more
    for c, d in ((2, 8), (3, 8), (4, 8), (2, 16), (3, 16), (4, 16)):
        if c == 2:
            bg, cols = ga_pairs[0], ga_pairs[1:256]
        else:
            bg, cols = many[0], many[1:256].copy()
            if c == 4:
                cols[:, 3] = 200
        out.append(("colour_257", "new", c, d, lambda h, w, c=c, d=d, bg=bg, cols=cols: _image(h, w, c, d, bg, [(FILL_AT, cols)]),
                    lambda im, p, k: _put(im, p, (7, 250, 9, 77))))
    return out


def edge_cases():
    """case 1: every (property, variant, class) at two widths for the properties with fewer than 8 variants, one width otherwise,
    with the deciding pixel at each of edge_positions"""
    variants = _edge_variants()
    cases = []
    per_prop = {}
    for v in variants:
        per_prop.setdefault(v[0], []).append(v)
    for prop, vs in per_prop.items():
        reps = 2 if len(vs) < 8 else 1
        k = 0
        for r in range(reps):
            for (_, var, c, d, build, change) in vs:
                w = WIDTHS[k % len(WIDTHS)]
                k += 1
                h, w = edge_shape(w)
                base = build(h, w)
                want = fmt_of(base)
                for j, (pos_name, p) in enumerate(edge_positions(h, w).items()):
                    changed = change(base, p, j)
                    cases.append(Case(f"{prop}_{var}_c{c}_d{d}_w{w}_{pos_name}", base, changed, p, want, fmt_of(changed), c, d,
                                      {"prop": prop, "w": w, "pos": pos_name}))
    return cases


# ---- case 2: the early stop ------------------------------------------------------------------------------------------------------
EARLY_ROWS = ("rgba8_rgb_vs_rgba", "rgba8_ga_vs_rgba", "rgba8_palette_vs_rgba", "rgb16_rgb8_vs_rgb16", "rgba16_rgba8_vs_rgba16",
              "rgba16_rgb16_vs_rgba16")
EARLY_BITS = {"rgba8_rgb_vs_rgba": (OVERFLOW | NOT_GRAY, NOT_OPAQUE), "rgba8_ga_vs_rgba": (OVERFLOW | NOT_OPAQUE, NOT_GRAY),
              "rgba8_palette_vs_rgba": (NOT_GRAY | NOT_OPAQUE, OVERFLOW), "rgb16_rgb8_vs_rgb16": (OVERFLOW | NOT_GRAY, NOT_REP8),
              "rgba16_rgba8_vs_rgba16": (OVERFLOW | NOT_GRAY | NOT_OPAQUE, NOT_REP8),
              "rgba16_rgb16_vs_rgba16": (OVERFLOW | NOT_GRAY | NOT_REP8, NOT_OPAQUE)}
EARLY_CLASS = {"rgba8_rgb_vs_rgba": (4, 8), "rgba8_ga_vs_rgba": (4, 8), "rgba8_palette_vs_rgba": (4, 8), "rgb16_rgb8_vs_rgb16": (3, 16),
               "rgba16_rgba8_vs_rgba16": (4, 16), "rgba16_rgb16_vs_rgba16": (4, 16)}
FAR = ("cta0_last_step", "cta0_last", "mid_cta_last_step", "last_cta_first", "last")
EARLY_SPAN = 2 * RED_THREADS                      # the early overflow colours fill each CTA's steps 0 and 1


def _early_base(row, h, w):
    c, d = EARLY_CLASS[row]
    n = h * w
    ctas = analyze_ctas(w, h)
    many = distinct_rgb(EARLY_SPAN, 11)
    if row == "rgba8_ga_vs_rgba":
        g = np.arange(EARLY_SPAN)
        many = np.stack([g % 256, g % 256, g % 256, 100 + g // 256], 1).astype(np.uint8)
    if row == "rgba16_rgba8_vs_rgba16":
        many[:, 3] = 128
    bg = {"rgba8_rgb_vs_rgba": (10, 20, 30, 255), "rgba8_ga_vs_rgba": (100, 100, 100, 255), "rgba8_palette_vs_rgba": (10, 20, 30, 128),
          "rgb16_rgb8_vs_rgb16": (10, 20, 30, 255), "rgba16_rgba8_vs_rgba16": (10, 20, 30, 128),
          "rgba16_rgb16_vs_rgba16": (10, 20, 30, 255)}[row]
    if row == "rgba8_palette_vs_rgba":
        cols = distinct_rgb(255, 12)
        cols[:, 3] = 128
        return _image(h, w, c, d, bg, [(FILL_AT, cols)])
    img = _image(h, w, c, d, bg, [(b * RED_PIXELS, many[:min(EARLY_SPAN, n - b * RED_PIXELS)]) for b in range(ctas)])
    if row == "rgba16_rgb16_vs_rgba16":
        img[..., 0] ^= 1                                           # every R sample off by one: not 8-bit representable anywhere
    return img


def _early_change(row, img, p):
    if row == "rgba8_rgb_vs_rgba":
        return _set(img, p, a=254)
    if row == "rgba8_ga_vs_rgba":
        return _set(img, p, r=int(img.reshape(-1, 4)[p, 0]) ^ 1)
    if row == "rgba8_palette_vs_rgba":
        return _set(img, p, r=201, g=202, b=203, a=204)
    if row == "rgb16_rgb8_vs_rgb16":
        return _set(img, p, g=int(img.reshape(-1, 3)[p, 1]) + 1)
    if row == "rgba16_rgba8_vs_rgba16":
        return _set(img, p, a=128 * 257 + 1)
    return _set(img, p, a=65534)


def early_stop_cases():
    """case 2: each row of the table in DESIGN §4.6 with its late evidence at each FAR position, at rotating widths"""
    cases, k = [], 0
    for row in EARLY_ROWS:
        c, d = EARLY_CLASS[row]
        for pos in FAR:
            h, w = edge_shape(WIDTHS[k % len(WIDTHS)])
            k += 1
            base = _early_base(row, h, w)
            p = edge_positions(h, w)[pos]
            changed = _early_change(row, base, p)
            cases.append(Case(f"early_{row}_w{w}_{pos}", base, changed, p, fmt_of(base), fmt_of(changed), c, d,
                              {"row": row, "pos": pos, "w": w}))
    return cases


def early_evidence_steps(img):
    """{CTA: [the evidence bits the CTA alone has read by the end of each of its steps]}"""
    h, w, c = img.shape
    flat = img.reshape(-1, c).astype(np.int64)
    out = {}
    for b in range(analyze_ctas(w, h)):
        seen, cols = 0, set()
        for s in range(RED_ITERS):
            px = flat[b * RED_PIXELS + s * RED_THREADS: b * RED_PIXELS + (s + 1) * RED_THREADS]
            if not len(px):
                break
            seen |= _evidence(px, c, img.dtype)
            cols |= set(key_of(_rgba8(px, c, img.dtype)).tolist())
            if len(cols) > 256:
                seen |= OVERFLOW
            out.setdefault(b, []).append(seen)
    return out


def _rgba8(px, c, dtype):
    v = px // 257 if dtype == np.uint16 else px
    r = v[:, 0]
    g, b = (r, r) if c <= 2 else (v[:, 1], v[:, 2])
    a = v[:, c - 1] if c in (2, 4) else np.full_like(r, 255)
    return np.stack([r, g, b, a], 1)


def _evidence(px, c, dtype):
    amax = 65535 if dtype == np.uint16 else 255
    bits = 0
    if dtype == np.uint16 and (px % 257 != 0).any():
        bits |= NOT_REP8
    if c in (2, 4) and (px[:, c - 1] != amax).any():
        bits |= NOT_OPAQUE
    if c >= 3 and ((px[:, 0] != px[:, 1]) | (px[:, 0] != px[:, 2])).any():
        bits |= NOT_GRAY
    return bits


# ---- case 3: colour-set edges ----------------------------------------------------------------------------------------------------
def colour_set_images():
    """[(name, image, intended (format, depth), facts)]"""
    out = []
    h, w = 3, RED_PIXELS                                   # three full CTAs, one row each
    zero = np.zeros(4, np.uint8)
    cols = distinct_rgb(256, 21)
    cols[:, 3] = np.arange(256) % 7 * 30                   # translucent, so the zero colour cannot be told from alpha alone
    for n_other, want in ((255, ("palette", 8)), (256, ("rgba", 8))):
        img = _image(h, w, 4, 8, cols[0], [(FILL_AT, cols[:n_other])])
        img.reshape(-1, 4)[-1] = zero                      # the zero colour at the last pixel only
        out.append((f"zero_last_k{n_other + 1}", img, want, {"K": n_other + 1, "zero_at": h * w - 1}))
    coll, slot = colliding_rgb(257)
    for n, want in ((256, ("palette", 8)), (257, ("rgb", 8))):
        one_cta = _image(h, w, 3, 8, coll[0], [(FILL_AT, coll[:n])])
        out.append((f"collide_{n}_one_cta", one_cta, want, {"K": n, "slot": slot, "keys": key_of(coll[:n])}))
        spread = _image(h, w, 3, 8, coll[0], [(b * RED_PIXELS + 1000, coll[b:n:3]) for b in range(3)])
        out.append((f"collide_{n}_three_ctas", spread, want, {"K": n, "slot": slot, "keys": key_of(coll[:n])}))
    for n, want in ((255, ("palette", 8)), (256, ("rgba", 8))):
        img = _image(h, w, 4, 8, coll[0], [(FILL_AT, coll[:n])])
        img.reshape(-1, 4)[FILL_AT + 2 * RED_PIXELS] = zero
        out.append((f"collide_{n}_and_zero", img, want, {"K": n + 1, "slot": slot, "keys": key_of(coll[:n])}))
    # one CTA alone sees 257 colours, the others one
    img = _image(h, w, 3, 8, cols[0], [(RED_PIXELS + 4000, distinct_rgb(257, 22))])
    out.append(("one_cta_257", img, ("rgb", 8), {"K": 257}))
    # 16-bit: high bytes take at most 256 values, the samples are not multiples of 257
    rng = np.random.default_rng(23)
    for c in (1, 3, 4):
        hi = distinct_rgb(200, 24)[rng.integers(0, 200, 64 * 64)][:, :c].astype(np.uint16)
        img = (hi << 8 | rng.integers(0, 256, hi.shape).astype(np.uint16)).reshape(64, 64, c)
        if c == 4:
            img[..., 3] = 0xFFFF
        out.append((f"hi_bytes_16_c{c}", img, ({1: "gray", 3: "rgb", 4: "rgb"}[c], 16), {"hi_colours": 200}))
    return out


def racing_same_colours(ctas=1024):
    """every CTA (one row of 8192 pixels) inserts the same 256 colours, starting at a different one and in either direction;
    pixel ids follow the palette order, so rows are ramps"""
    pal = np.sort(key_of(distinct_rgb(256, 31)))
    cols = np.stack([pal >> 24, (pal >> 16) & 255, (pal >> 8) & 255], 1).astype(np.uint8)
    x = np.arange(RED_PIXELS)
    r = np.arange(ctas)[:, None]
    ids = np.where(r % 2 == 0, x + 37 * r, 37 * r - x) % 256
    return cols[ids]


def overflow_16k_colours(chans, ctas=64):
    """64 CTAs (rows) each with 256 distinct colours of their own, 16384 in all"""
    k = np.arange(ctas * 256, dtype=np.int64) * 977 + 5
    cols = np.stack([(k >> 16) & 255, (k >> 8) & 255, k & 255, 60 + k % 190], 1).astype(np.uint8)[:, :chans]
    x = np.arange(RED_PIXELS)
    r = np.arange(ctas)[:, None]
    return cols[r * 256 + (x * 5 + r) % 256]


# ---- case 4: the rule sweep ------------------------------------------------------------------------------------------------------
SWEEP_K = (1, 2, 3, 4, 5, 16, 17, 255, 256, 257)


def sweep_images():
    """[(name, image, intent)]: per class, small images over K (with and without the zero colour), gray / not, opaque / 0, 1 or all
    translucent palette entries, lattice depths and representable / not; realisable combinations only (the CPU test checks each
    intent against reduce_model.analyse)"""
    out = []
    h, w = 11, 29
    for c, d in CLASSES:
        grays = (True,) if c <= 2 else (True, False)
        alphas = ("opaque",) if c in (1, 3) else ("opaque", "one", "all")
        reps = (True,) if d == 8 else (True, False)
        for K in SWEEP_K:
            for gray in grays:
                for al in alphas:
                    for zero in ((False, True) if c in (2, 4) and al != "opaque" else (False,)):
                        for rep in reps:
                            img = _sweep_image(h, w, c, d, K, gray, al, zero, rep)
                            if img is not None:
                                out.append((f"c{c}_d{d}_K{K}_{'gray' if gray else 'rgb'}_{al}{'_zero' if zero else ''}"
                                            f"{'' if rep else '_not_rep8'}", img,
                                            {"K": K, "gray": gray, "alpha": al, "zero": zero, "rep8": rep}))
        # the lattice depths of gray opaque images
        for dd in (1, 2, 4):
            lv = np.arange(0, 256, 255 // ((1 << dd) - 1))
            for K in (1, len(lv)):
                cols = np.array([[g, g, g, 255] for g in lv[:K][::-1]], np.uint8)
                img = _fill_cycle(h, w, c, d, cols)
                out.append((f"c{c}_d{d}_lattice{dd}_K{K}", img, {"K": K, "gray": True, "alpha": "opaque", "zero": False,
                                                                  "rep8": True, "lattice": dd if K > 1 or lv[0] else 1}))
    return out


def _fill_cycle(h, w, c, d, cols):
    """every colour of cols at least once, in a scattered order"""
    n = h * w
    assert n >= len(cols)
    return as_class(cols[(np.arange(n) * 7) % len(cols)], c, d).reshape(h, w, c)


def _sweep_image(h, w, c, d, K, gray, al, zero, rep):
    """K distinct colours: gray (g, g, g) or not; alpha 255, one translucent entry or all translucent; the zero colour among the
    translucent ones; at 16 bits, one sample off by one (its high byte, and so K, unchanged).  None when not realisable."""
    if K > 256 and (c == 1 or (gray and al == "opaque")):
        return None                                            # at most 256 gray levels without an alpha to tell them apart
    if zero and al == "opaque":
        return None
    i = np.arange(K)
    if gray:
        rgba = np.stack([i % 256, i % 256, i % 256, np.where(i < 256, 255, 254)], 1)
    else:
        rgba = distinct_rgb(K, K + 1000 * c).astype(np.int64)
    if al == "one":
        rgba[-1, 3] = 254 if K > 256 else 100
        if zero:
            rgba[-1] = 0
    elif al == "all":
        rgba[:, 3] = 10 + i % 200 if not (gray and K > 256) else np.where(i < 256, 20, 21)
        if zero:
            rgba[0] = 0
    if len(np.unique(key_of(rgba.astype(np.uint8)))) != K or (not gray and (rgba[:, 0] == rgba[:, 1]).all() and
                                                                  (rgba[:, 1] == rgba[:, 2]).all()):
        return None                                            # e.g. K = 1 of the zero colour only: gray after all
    img = _fill_cycle(h, w, c, d, rgba.astype(np.uint8))
    if not rep:
        img[0, 0, :1 if c <= 2 else 3] ^= 1                            # R (and G, B alike): gray stays gray, alpha untouched
    return img


# ---- case 5: conversion widths ---------------------------------------------------------------------------------------------------
CONV_WIDTHS = range(1, 68)


def conversion_modes():
    """{mode: (chans, depth, colours builder K -> [K, 4] RGBA or None, intended (format, depth))}"""
    pal = distinct_rgb(256, 41)
    gray_many = np.stack([np.arange(256)] * 3 + [np.full(256, 255)], 1).astype(np.uint8)
    ga_many = np.stack([np.arange(300) % 256] * 3 + [100 + np.arange(300) // 256], 1).astype(np.uint8)
    rgba_op = distinct_rgb(300, 42)
    modes = {}
    for bits, K in ((1, 2), (2, 4), (4, 16), (8, 256)):
        modes[f"palette{bits}_from_rgb8"] = (3, 8, pal[:K], ("palette", bits))
        modes[f"palette{bits}_from_rgba16"] = (4, 16, pal[:K], ("palette", bits))
    for bits in (1, 2, 4):
        lv = np.arange(0, 256, 255 // ((1 << bits) - 1))
        cols = np.array([[g, g, g, 255] for g in lv], np.uint8)
        modes[f"gray{bits}_from_gray8"] = (1, 8, cols, ("gray", bits))
        modes[f"gray{bits}_from_rgb16"] = (3, 16, cols, ("gray", bits))
    modes["gray8_from_rgb8"] = (3, 8, gray_many, ("gray", 8))
    modes["gray8_from_ga8"] = (2, 8, gray_many, ("gray", 8))
    modes["ga8_from_rgba8"] = (4, 8, ga_many, ("ga", 8))
    modes["rgb8_from_rgba8"] = (4, 8, rgba_op, ("rgb", 8))
    modes["gray8_from_gray16"] = (1, 16, gray_many, ("gray", 8))
    modes["ga8_from_ga16"] = (2, 16, ga_many, ("ga", 8))
    modes["rgb8_from_rgb16"] = (3, 16, rgba_op, ("rgb", 8))
    modes["rgba8_from_rgba16"] = (4, 16, np.concatenate([rgba_op[:, :3], np.full((300, 1), 9)], 1), ("rgba", 8))
    modes["rgb16_from_rgba16"] = (4, 16, None, ("rgb", 16))
    modes["ga16_from_rgba16"] = (4, 16, None, ("ga", 16))
    return modes


def conversion_image(mode, w, h=None, seed=0):
    """an image of the mode at width w; its rows hold every colour of the mode (so K and the format do not depend on w) unless
    h is given"""
    c, d, cols, _ = conversion_modes()[mode]
    rng = np.random.default_rng(seed * 1000 + w)
    if cols is None:
        h = h or 5
        img = rng.integers(0, 65536, (h, w, 4)).astype(np.uint16)
        if mode == "rgb16_from_rgba16":
            img[..., 3] = 65535
        else:
            img[..., 1] = img[..., 0]
            img[..., 2] = img[..., 0]
        return img
    K = len(cols)
    h = h or max(3, -(-K // w))
    idx = rng.permutation(np.arange(h * w) % K) if h * w >= K else rng.integers(0, K, h * w)
    return as_class(cols[idx], c, d).reshape(h, w, c)


def mode_words(mode, w):
    fmt, depth = conversion_modes()[mode][3]
    bits = {"gray": 1, "ga": 2, "rgb": 3, "rgba": 4}.get(fmt, 1) * depth
    return conv_words(w, fmt, bits, depth)


def cta_shapes(mode):
    """[(w, h, words * h)] for words * h nearest 255, 256 and 257 (one conversion CTA, exactly full, one word into a second), with
    room for every colour of the mode"""
    cols = conversion_modes()[mode][2]
    K = 1 if cols is None else len(cols)
    out = []
    for target in (CONV_THREADS - 1, CONV_THREADS, CONV_THREADS + 1):
        best = None
        for w in CONV_WIDTHS:
            words = mode_words(mode, w)
            for h in (target // words, -(-target // words)):
                if h >= 1 and h * w >= K:
                    cand = (abs(words * h - target), w, h, words * h)
                    best = cand if best is None or cand < best else best
        out.append(best[1:])
    return out


# ---- case 6: image boundaries in one call ----------------------------------------------------------------------------------------
BOUNDARY_PIXELS = (1, 8191, 8192, 8193, 16385)


def boundary_images():
    """[(name, image)]: images of BOUNDARY_PIXELS pixels (one row each), mixed in one call.  The even ones are RGBA8 with their own
    200 colours (1000 over the call, under 256 per image) that become palettes, the first and the last pixel each a colour of
    its own; the odd ones are gray8 images on the 4-bit lattice but for the first pixel (1) and the last (254), so that they
    keep their format and are read in place"""
    out = []
    for i, n in enumerate(BOUNDARY_PIXELS):
        if i % 2 == 0:
            cols = distinct_rgb(202, 50 + i)
            cols[:, 3] = 40 + i
            img = cols[2 + np.arange(n) % 200].reshape(1, n, 4).copy()
            img[0, 0] = cols[0]
            img[0, -1] = cols[1] if n > 1 else cols[0]
            out.append((f"px{n}_change", img))
        else:
            img = (np.arange(n) % 16 * 17).astype(np.uint8).reshape(1, n, 1)
            img[0, 0], img[0, -1] = 1, 254
            out.append((f"px{n}_keep", img))
    return out
