// fpng_b200/csrc/reduce_kernels.cu -- sm_90a kernels of the colour-type reduction (FPNGB_ENCODE_REDUCE, DESIGN §4.6 "Colour-type
// reduction"): the analysis that decides which formats hold an image exactly, the palette finalise, and the conversion pre-pass
// that writes the reduced rows.
//
// Analysis: a CTA reads kRedPixels consecutive pixels (row-major) of one image, 256 threads one pixel apart.  Each thread ORs its
// negative evidence (kRed* flags) and a warp publishes it with one atomicOr; each thread inserts its pixel's colour into a CTA-local
// shared set, merged into the image's global ReduceTable when the CTA ends.  A CTA stops reading once its image is decided negative
// on every property that can still change the format (kRedOverflow, kRedNotGray for 3 and 4 channels, kRedNotOpaque with an alpha,
// kRedNotRep8 for 16 bits), so an RGB photo costs a fraction of one read.
//
// The sets hash a key k to slot (k * 0x9E3779B1) >> 23 (the top 9 bits of the product), probing linearly.  A slot holding 0 is empty,
// so the colour 0x00000000 sets kRedHasZero instead of taking a slot.  Both sets stop at 257 colours (kRedOverflow); each has 512
// slots, so a probe always ends within 512 steps even while CTAs race past the 257th insert.
#include "kernels.cuh"

namespace fpngb {

constexpr uint32_t kRedThreads = 256, kRedIters = 32, kRedPixels = kRedThreads * kRedIters;
constexpr uint32_t kRedConvThreads = 256;

uint32_t reduce_analyze_ctas(uint32_t w, uint32_t h) { return (uint32_t)(((unsigned long long)w * h + kRedPixels - 1) / kRedPixels); }
uint32_t reduce_convert_ctas(uint32_t words, uint32_t h)
{
    return (uint32_t)(((unsigned long long)words * h + kRedConvThreads - 1) / kRedConvThreads);
}

__device__ __forceinline__ uint32_t red_hash(uint32_t key) { return (key * 0x9E3779B1u) >> 23; }

// Inserts key into the set (keys[512], count, the kRedHasZero bit of *zero_flags).  False when the set now holds 257 or more colours
// or could not take the key: the caller sets kRedOverflow.
__device__ bool red_insert(uint32_t* keys, uint32_t* count, uint32_t* zero_flags, uint32_t key)
{
    if (key == 0u) {
        if (atomicOr(zero_flags, kRedHasZero) & kRedHasZero) return true;
        return atomicAdd(count, 1u) < 256u;
    }
    volatile uint32_t* vk = keys;
    uint32_t s = red_hash(key);
    for (uint32_t probe = 0; probe < kReduceSlots; probe++, s = (s + 1u) & (kReduceSlots - 1u)) {
        uint32_t cur = vk[s];
        if (cur == 0u) {
            cur = atomicCAS(&keys[s], 0u, key);
            if (cur == 0u) return atomicAdd(count, 1u) < 256u;
        }
        if (cur == key) return true;
    }
    return false;
}

template <class T>
__device__ __forceinline__ uint32_t red_sample(const uint8_t* q) { return (uint32_t)__ldg(reinterpret_cast<const T*>(q)); }

// The four samples (R, G, B, A at full depth; alpha `amax` when absent) of pixel (x, y)
template <class T>
__device__ __forceinline__ void red_pixel(const ReduceDesc& d, uint32_t x, uint32_t y, uint32_t v[4], uint32_t amax)
{
    const uint8_t* q = d.src + (unsigned long long)y * d.row + (unsigned long long)x * d.pixel;
    v[0] = red_sample<T>(q);
    if (d.chans >= 3) { v[1] = red_sample<T>(q + d.chan); v[2] = red_sample<T>(q + 2 * d.chan); }
    else { v[1] = v[0]; v[2] = v[0]; }
    v[3] = (d.chans == 2 || d.chans == 4) ? red_sample<T>(q + (d.chans - 1) * d.chan) : amax;
}

// 8-bit value of a sample (v >> 8 is v / 257 for the multiples of 257, the only 16-bit samples whose 8-bit value is used)
__device__ __forceinline__ uint32_t red_key(const uint32_t v[4], uint32_t shift)
{
    return (v[0] >> shift) << 24 | (v[1] >> shift) << 16 | (v[2] >> shift) << 8 | (v[3] >> shift);
}

template <class T>
__device__ void reduce_analyze_image(const ReduceParams& p, const ReduceDesc& d, uint32_t img, unsigned long long p0, uint32_t* skeys,
                                     uint32_t* scount, uint32_t* sflags)
{
    constexpr uint32_t shift = sizeof(T) == 2 ? 8u : 0u, amax = sizeof(T) == 2 ? 0xFFFFu : 0xFFu;
    ReduceState* st = p.st + img;
    volatile uint32_t* gflags = &st->flags;
    // the evidence that can still change the format; every bit set: nothing left to learn
    const uint32_t need = kRedOverflow | kRedNotGray | ((d.chans & 1u) ? 0u : kRedNotOpaque) | (sizeof(T) == 2 ? kRedNotRep8 : 0u);
    const unsigned long long total = (unsigned long long)d.w * d.h;
    unsigned long long pix = p0 + threadIdx.x;
    uint32_t y = (uint32_t)(pix / d.w), x = (uint32_t)(pix - (unsigned long long)y * d.w);
    const uint32_t dy = kRedThreads / d.w, dx = kRedThreads % d.w;
    for (uint32_t it = 0; it < kRedIters && pix < total; it++, pix += kRedThreads) {
        const uint32_t g = *gflags;
        if ((g & need) == need) break;
        uint32_t v[4];
        red_pixel<T>(d, x, y, v, amax);
        uint32_t mine = 0;
        if (sizeof(T) == 2) {
#pragma unroll
            for (int c = 0; c < 4; c++) if ((v[c] >> 8) != (v[c] & 0xFFu)) mine |= kRedNotRep8;
        }
        if (v[3] != amax) mine |= kRedNotOpaque;
        if (v[0] != v[1] || v[0] != v[2]) mine |= kRedNotGray;
        const uint32_t g8 = v[0] >> shift;
        mine |= g8 % 17u ? kRedNotL4 | kRedNotL2 | kRedNotL1 : g8 % 85u ? kRedNotL2 | kRedNotL1 : g8 % 255u ? kRedNotL1 : 0u;
        if (!(g & kRedOverflow) && !red_insert(skeys, scount, sflags, red_key(v, shift))) mine |= kRedOverflow;
        const uint32_t active = __activemask();
        const uint32_t any = __reduce_or_sync(active, mine);
        if ((any & ~g) && (threadIdx.x & 31u) == (uint32_t)__ffs(active) - 1u) atomicOr(&st->flags, any);
        y += dy; x += dx;
        if (x >= d.w) { x -= d.w; y++; }
    }
    __syncthreads();
    // merge the CTA's colours into the image's set
    if (*gflags & kRedOverflow) return;
    ReduceTable* tab = p.tab + img;
    bool over = false;
    for (uint32_t s = threadIdx.x; s < kReduceSlots && !over; s += kRedThreads)
        if (skeys[s] && !red_insert(tab->key, &st->count, &st->flags, skeys[s])) over = true;
    if (threadIdx.x == 0 && (*sflags & kRedHasZero) && !red_insert(tab->key, &st->count, &st->flags, 0u)) over = true;
    if (over) atomicOr(&st->flags, kRedOverflow);
}

__global__ void __launch_bounds__(kRedThreads) reduce_analyze_kernel(ReduceParams p)
{
    __shared__ uint32_t skeys[kReduceSlots];
    __shared__ uint32_t scount, sflags;
    uint32_t lo = 0, hi = p.count - 1;
    const unsigned long long b = blockIdx.x;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (p.desc[mid].cta_start <= b) lo = mid; else hi = mid - 1;
    }
    const ReduceDesc& d = p.desc[lo];
    for (uint32_t s = threadIdx.x; s < kReduceSlots; s += kRedThreads) skeys[s] = 0u;
    if (threadIdx.x == 0) { scount = 0u; sflags = 0u; }
    __syncthreads();
    const unsigned long long p0 = (b - d.cta_start) * kRedPixels;
    if (d.elem == 2) reduce_analyze_image<uint16_t>(p, d, lo, p0, skeys, &scount, &sflags);
    else reduce_analyze_image<uint8_t>(p, d, lo, p0, skeys, &scount, &sflags);
}

// One CTA per image: the colours of the set in palette order -- first the entries with alpha below 255 ascending by their key, then
// the opaque ones ascending by RGB (= by key) -- as ReduceResult::pal, and each colour's index in ReduceTable::index (the zero colour's
// in ReduceState::zero_index).  Sort key: opaque << 42 | colour << 10 | slot (slot 512: the zero colour), bitonic over 256 entries.
__global__ void __launch_bounds__(256) reduce_finalise_kernel(ReduceParams p)
{
    __shared__ unsigned long long sk[256];
    __shared__ uint32_t n;
    const uint32_t img = blockIdx.x, t = threadIdx.x;
    ReduceState* st = p.st + img;
    ReduceTable* tab = p.tab + img;
    ReduceResult* res = p.res + img;
    const uint32_t flags = st->flags, count = st->count;
    if (t == 0) { res->flags = flags; res->count = count; n = 0; }
    if (flags & kRedOverflow) return;                                     // uniform across the CTA
    sk[t] = ~0ull;
    __syncthreads();
    for (uint32_t s = t; s <= kReduceSlots; s += 256) {
        const uint32_t k = s < kReduceSlots ? tab->key[s] : 0u;
        if (s < kReduceSlots ? k != 0u : (flags & kRedHasZero) != 0u) {
            const uint32_t at = atomicAdd(&n, 1u);
            sk[at] = (unsigned long long)((k & 0xFFu) == 0xFFu) << 42 | (unsigned long long)k << 10 | s;
        }
    }
    __syncthreads();
    for (uint32_t k = 2; k <= 256; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            const uint32_t o = t ^ j;
            if (o > t) {
                const unsigned long long a = sk[t], c = sk[o];
                if (((t & k) == 0) == (a > c)) { sk[t] = c; sk[o] = a; }
            }
            __syncthreads();
        }
    if (t < n) {
        const unsigned long long e = sk[t];
        const uint32_t slot = (uint32_t)(e & 1023u);
        res->pal[t] = (uint32_t)(e >> 10);
        if (slot == kReduceSlots) st->zero_index = t; else tab->index[slot] = (uint8_t)t;
    }
}

void launch_reduce_analyze(const ReduceParams& p, unsigned long long total_ctas, cudaStream_t s)
{
    reduce_analyze_kernel<<<(uint32_t)total_ctas, kRedThreads, 0, s>>>(p);
    reduce_finalise_kernel<<<p.count, 256, 0, s>>>(p);
}

// palette index of a colour key (present in the set by construction)
__device__ __forceinline__ uint32_t red_lookup(const ReduceConvDesc& d, uint32_t key)
{
    if (key == 0u) return d.st->zero_index;
    uint32_t s = red_hash(key);
    while (__ldg(&d.tab->key[s]) != key) s = (s + 1u) & (kReduceSlots - 1u);
    return __ldg(&d.tab->index[s]);
}

template <class T>
__device__ uint32_t reduce_word(const ReduceConvDesc& d, uint32_t y, uint32_t k)
{
    constexpr uint32_t shift = sizeof(T) == 2 ? 8u : 0u;
    const uint8_t* row = d.src + (unsigned long long)y * d.row;
    uint32_t word = 0;
    if (d.mode < 2) {                                                     // packed, MSB-first: pixel j at bit 8*byte + 8 - bits - off
        const uint32_t per = 32u / d.bits, x0 = k * per;
        for (uint32_t j = 0; j < per && x0 + j < d.w; j++) {
            const uint8_t* q = row + (unsigned long long)(x0 + j) * d.pixel;
            uint32_t v;
            if (d.mode == 0) {
                uint32_t s[4];
                s[0] = red_sample<T>(q);
                if (d.chans >= 3) { s[1] = red_sample<T>(q + d.chan); s[2] = red_sample<T>(q + 2 * d.chan); }
                else { s[1] = s[0]; s[2] = s[0]; }
                s[3] = (d.chans == 2 || d.chans == 4) ? red_sample<T>(q + (d.chans - 1) * d.chan) : (sizeof(T) == 2 ? 0xFFFFu : 0xFFu);
                v = red_lookup(d, red_key(s, shift));
            } else {
                v = (red_sample<T>(q) >> shift) / d.step;
            }
            const uint32_t bit = j * d.bits;
            word |= v << (8 * (bit >> 3) + 8 - d.bits - (bit & 7));
        }
    } else {                                                              // tight samples, little-endian bytes
        const uint32_t oc = d.bits, ob = d.out_bytes, row_bytes = d.w * oc * ob;
        for (uint32_t i = 0; i < 4; i++) {
            const uint32_t byte = 4 * k + i;
            if (byte >= row_bytes) break;
            const uint32_t s = byte / ob, x = s / oc, j = s - x * oc;
            const uint32_t c = (oc == 2 && j == 1) ? d.chans - 1 : j;
            const uint32_t v = red_sample<T>(row + (unsigned long long)x * d.pixel + c * d.chan);
            const uint32_t b = ob == 2 ? (v >> (8 * (byte & 1u))) & 0xFFu : v >> shift;
            word |= b << (8 * i);
        }
    }
    return word;
}

__global__ void __launch_bounds__(kRedConvThreads) reduce_convert_kernel(ReduceConvParams p)
{
    uint32_t lo = 0, hi = p.count - 1;
    const unsigned long long b = blockIdx.x;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (p.desc[mid].cta_start <= b) lo = mid; else hi = mid - 1;
    }
    const ReduceConvDesc& d = p.desc[lo];
    const unsigned long long g = (b - d.cta_start) * kRedConvThreads + threadIdx.x;    // output word of the image
    if (g >= (unsigned long long)d.words * d.h) return;
    const uint32_t y = (uint32_t)(g / d.words), k = (uint32_t)(g - (unsigned long long)y * d.words);
    const uint32_t v = d.elem == 2 ? reduce_word<uint16_t>(d, y, k) : reduce_word<uint8_t>(d, y, k);
    reinterpret_cast<uint32_t*>(p.dst + d.dst + (unsigned long long)y * 4ull * d.words)[k] = v;
}

void launch_reduce_convert(const ReduceConvParams& p, unsigned long long total_ctas, cudaStream_t s)
{
    reduce_convert_kernel<<<(uint32_t)total_ctas, kRedConvThreads, 0, s>>>(p);
}

}  // namespace fpngb
