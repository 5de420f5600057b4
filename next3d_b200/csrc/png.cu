// PNG encoder for batches of uint8 RGB images (next3d_b200/png.py; DESIGN.md section 3.6).  Every decision is integer arithmetic
// on one image's pixels, so the bytes depend on nothing else (not the batch, the grid or the device):
//   png_filter_rows    one warp per row: the filter (0-4) of least sum of |int8(filtered byte)|, ties to the lower number, and
//                      the filtered row (filter byte first) into scratch.
//   png_deflate        one warp per stripe of stripe_rows(W) rows: a greedy LZ77 parse over fixed candidate distances (the
//                      previous byte, pixel and second pixel, the byte above, the pixels above-left and above-right; matches may
//                      reach into earlier stripes), one dynamic-Huffman block (codes limited to 15 / 7 bits by halving the
//                      frequencies), or stored blocks when those are no larger.  Every stripe but the last ends with an empty
//                      stored block, so that the stripes' bit streams concatenate with a byte copy.
//   png_layout         one block per image: stripe offsets, the chunk headers, the zlib header and the Adler-32 trailer.
//   png_copy_stripes   one block per stripe: its bytes into the file.
//   png_crc_segments   one thread per 4096-byte segment of the IDAT chunk: the segment's CRC from a zero register.
//   png_crc_finish     one thread per image: the segments combined (crc * x^(8 len) mod P + segment), IDAT's CRC and IEND.
// The numpy restatement in tests/png_oracle.py makes the same decisions and writes the same bytes.
#include "common.cuh"

namespace {

constexpr int kStripeBytes = 32768;       // target filtered bytes per stripe
constexpr int kMaxDist = 32768;
constexpr int kMaxMatch = 258;
constexpr int kStoredMax = 65535;
constexpr int kCrcSegment = 4096;
constexpr int kCands = 6;
constexpr int kWarps = 4;                 // warps (stripes) per png_deflate block
constexpr int kHeadBytes = 8 + 25 + 8 + 2;          // signature, IHDR chunk, IDAT length and type, zlib header
constexpr int kTailBytes = 4 + 4 + 12;              // Adler-32, IDAT CRC, IEND chunk
constexpr uint32_t kMatchFlag = 0x80000000u;        // token: literal byte, or kMatchFlag | length << 16 | distance

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                        131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                         2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct Geom {
    int n, H, W;
    int bpr;              // bytes per filtered row, 3W + 1
    int rows;             // rows per stripe
    int stripes;          // per image
    int64_t raw;          // filtered bytes per image, H * bpr
    int64_t stripe_cap;   // bytes of a stripe's output slot: stored size of a full stripe, rounded up to 8
    int64_t cap;          // file capacity
    int nseg;             // CRC segments per image, at most
    int dist[kCands];     // candidate distances, 0 = unused
    // scratch, per image
    uint8_t* flt;         // [n][raw]
    uint32_t* tok;        // [n][raw]
    uint8_t* sbuf;        // [n][stripes][stripe_cap]
    int64_t* ssize;       // [n][stripes]: bytes of each stripe, then (png_layout) their offsets in the zlib stream
    uint32_t* crc;        // [n][nseg]
    int64_t* body;        // [n]: bytes of all stripes
};

__host__ __device__ inline int64_t stored_bytes(int64_t n) { return n + 5 * ((n + kStoredMax - 1) / kStoredMax); }
inline int64_t align(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

int make_geom(int n, int height, int width, Geom& g) {
    N3D_CHECK_ARG(n > 0 && height > 0 && width > 0 && width <= (1 << 24), "n3d_png: need n, height, width > 0 and width <= 2^24, got %d, %d, %d",
                  n, height, width);
    g.n = n;
    g.H = height;
    g.W = width;
    g.bpr = 3 * width + 1;
    g.rows = g.bpr >= kStripeBytes ? 1 : kStripeBytes / g.bpr;
    g.stripes = n3d_div_up(height, g.rows);
    g.raw = (int64_t)height * g.bpr;
    g.stripe_cap = align(stored_bytes((int64_t)g.rows * g.bpr), 8);
    const int64_t full = height / g.rows, last = height % g.rows;
    const int64_t body = full * stored_bytes((int64_t)g.rows * g.bpr) + (last ? stored_bytes(last * g.bpr) : 0);
    g.cap = kHeadBytes + body + kTailBytes;
    N3D_CHECK_ARG(g.cap - 8 - 25 - 12 - 12 <= 0x7fffffffLL, "n3d_png: a %dx%d image may exceed the 2^31 - 1 bytes of one IDAT chunk", height,
                  width);
    g.nseg = (int)((4 + g.cap - kHeadBytes + 2 + 4 + kCrcSegment - 1) / kCrcSegment);
    const int d[kCands] = {1, 3, 6, g.bpr, g.bpr - 3, g.bpr + 3};
    for (int k = 0; k < kCands; ++k) g.dist[k] = d[k] >= 1 && d[k] <= kMaxDist ? d[k] : 0;
    return N3D_OK;
}

// scratch layout: flt, tok, sbuf, ssize, crc, body (each 256-byte aligned)
int64_t layout(Geom& g, uint8_t* base) {
    int64_t o = 0;
    auto take = [&](int64_t bytes) { uint8_t* p = base ? base + o : nullptr; o += align(bytes, 256); return p; };
    g.flt = take(g.n * g.raw);
    g.tok = (uint32_t*)take(4 * g.n * g.raw);
    g.sbuf = take((int64_t)g.n * g.stripes * g.stripe_cap);
    g.ssize = (int64_t*)take(8LL * g.n * g.stripes);
    g.crc = (uint32_t*)take(4LL * g.n * g.nseg);
    g.body = (int64_t*)take(8LL * g.n);
    return o;
}

// ------------------------------------------------------------------------------------------------------------- filters
__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ uint32_t filtered(int f, int x, int a, int b, int c) {
    const int p = f == 0 ? 0 : f == 1 ? a : f == 2 ? b : f == 3 ? (a + b) >> 1 : paeth(a, b, c);
    return (uint32_t)(x - p) & 0xff;
}

__global__ void __launch_bounds__(128) png_filter_rows(const uint8_t* __restrict__ rgb, Geom g) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= (int64_t)g.n * g.H) return;
    const int y = (int)(r % g.H), rb = 3 * g.W;
    const uint8_t* cur = rgb + r * rb;
    const uint8_t* up = y ? cur - rb : nullptr;
    uint32_t cost[5] = {0, 0, 0, 0, 0};
    for (int x = lane; x < rb; x += 32) {
        const int v = cur[x], a = x >= 3 ? cur[x - 3] : 0, b = up ? up[x] : 0, c = (up && x >= 3) ? up[x - 3] : 0;
#pragma unroll
        for (int f = 0; f < 5; ++f) {
            const uint32_t t = filtered(f, v, a, b, c);
            cost[f] += t < 128 ? t : 256 - t;
        }
    }
    int best = 0;
    uint32_t bc = 0;
#pragma unroll
    for (int f = 0; f < 5; ++f) {
        uint32_t s = cost[f];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (f == 0 || s < bc) best = f, bc = s;
    }
    uint8_t* out = g.flt + (r / g.H) * g.raw + (int64_t)y * g.bpr;
    if (lane == 0) out[0] = (uint8_t)best;
    for (int x = lane; x < rb; x += 32) {
        const int v = cur[x], a = x >= 3 ? cur[x - 3] : 0, b = up ? up[x] : 0, c = (up && x >= 3) ? up[x - 3] : 0;
        out[1 + x] = (uint8_t)filtered(best, v, a, b, c);
    }
}

// ------------------------------------------------------------------------------------------------------------- Huffman
struct HuffWork {
    uint32_t f[286];        // working frequencies
    uint32_t w[2 * 286];    // node weights: sorted leaves, then internal nodes
    uint16_t parent[2 * 286];
    uint16_t sym[286];      // leaves in (frequency, symbol) order
    uint8_t depth[2 * 286];
};

struct StripeSmem {
    uint32_t lf[286], df[30], cf[19];
    uint8_t ll[286], dl[30], cl[19];
    uint16_t lc[286], dc[30], cc[19];
    uint16_t cls[286 + 30];         // code-length symbols: symbol | extra << 5
    HuffWork hw;
};

// Code lengths (at most `limit` bits) of the nonzero frequencies freq[0..n): Huffman's construction over leaves sorted by
// (frequency, symbol) with a leaf queue and a node queue (a leaf first on equal weights); at least two symbols get codes
// (symbols 0, then 1, get a count of 1 while fewer than two are used); while a code is too long, every nonzero frequency f
// becomes (f + 1) / 2.  Whole warp.
__device__ void limited_lengths(const uint32_t* freq, int n, int limit, uint8_t* len, HuffWork& h) {
    const int lane = threadIdx.x & 31;
    if (lane == 0) {
        int used = 0;
        for (int s = 0; s < n; ++s) h.f[s] = freq[s], used += freq[s] != 0;
        for (int s = 0; s < 2 && used < 2; ++s)
            if (!h.f[s]) h.f[s] = 1, ++used;
    }
    __syncwarp();
    while (true) {
        int m = 0;
        for (int s = 0; s < n; ++s) m += h.f[s] != 0;
        for (int s = lane; s < n; s += 32) {                      // rank of each used symbol in (frequency, symbol) order
            const uint32_t fs = h.f[s];
            if (!fs) continue;
            int rank = 0;
            for (int t = 0; t < n; ++t) {
                const uint32_t ft = h.f[t];
                rank += ft && (ft < fs || (ft == fs && t < s));
            }
            h.sym[rank] = (uint16_t)s;
            h.w[rank] = fs;
        }
        __syncwarp();
        int maxd = 0;
        if (lane == 0) {
            int i = 0, j = m;
            for (int k = m; k < 2 * m - 1; ++k) {
                int kid[2];
                for (int q = 0; q < 2; ++q) {
                    if (i < m && (j >= k || h.w[i] <= h.w[j])) kid[q] = i++;
                    else kid[q] = j++;
                }
                h.w[k] = h.w[kid[0]] + h.w[kid[1]];
                h.parent[kid[0]] = h.parent[kid[1]] = (uint16_t)k;
            }
            h.depth[2 * m - 2] = 0;
            for (int k = 2 * m - 3; k >= 0; --k) h.depth[k] = h.depth[h.parent[k]] + 1;
            for (int s = 0; s < n; ++s) len[s] = 0;
            for (int k = 0; k < m; ++k) {
                len[h.sym[k]] = h.depth[k];
                maxd = max(maxd, (int)h.depth[k]);
            }
            if (maxd > limit)
                for (int s = 0; s < n; ++s) h.f[s] = (h.f[s] + 1) >> 1;
        }
        maxd = __shfl_sync(0xffffffffu, maxd, 0);
        __syncwarp();
        if (maxd <= limit) return;
    }
}

// Canonical codes, bit-reversed for least-significant-bit-first output.  One thread.
__device__ void canonical_codes(const uint8_t* len, int n, uint16_t* code) {
    int bl[16] = {0}, nxt[16];
    for (int s = 0; s < n; ++s) bl[len[s]]++;
    bl[0] = 0;
    int c = 0;
    for (int b = 1; b < 16; ++b) {
        c = (c + bl[b - 1]) << 1;
        nxt[b] = c;
    }
    for (int s = 0; s < n; ++s)
        if (len[s]) code[s] = (uint16_t)(__brev((uint32_t)nxt[len[s]]++) >> (32 - len[s]));
}

__device__ __forceinline__ int len_sym(int len) {
    int k = 28;
    while (c_len_base[k] > len) --k;
    return k;
}

__device__ __forceinline__ int dist_sym(int d) {
    int k = 29;
    while (c_dist_base[k] > d) --k;
    return k;
}

// Bits of a token: its codes and extra bits in stream order (at most 15 + 5 + 15 + 13 = 48).
__device__ __forceinline__ uint64_t token_bits(uint32_t t, const StripeSmem& S, int& nb) {
    if (!(t & kMatchFlag)) {
        nb = S.ll[t];
        return S.lc[t];
    }
    const int len = (t >> 16) & 0x1ff, d = t & 0xffff, ls = len_sym(len), ds = dist_sym(d);
    uint64_t v = S.lc[257 + ls];
    int n = S.ll[257 + ls];
    v |= (uint64_t)(len - c_len_base[ls]) << n;
    n += c_len_extra[ls];
    v |= (uint64_t)S.dc[ds] << n;
    n += S.dl[ds];
    v |= (uint64_t)(d - c_dist_base[ds]) << n;
    nb = n + c_dist_extra[ds];
    return v;
}

// OR `nb` (<= 58) bits of v into the zeroed bit buffer at bit `pos`.
__device__ __forceinline__ void put_bits(unsigned long long* words, int64_t pos, uint64_t v, int nb) {
    if (!nb) return;
    const int o = (int)(pos & 63);
    atomicOr(words + (pos >> 6), (unsigned long long)(v << o));
    if (o + nb > 64) atomicOr(words + (pos >> 6) + 1, (unsigned long long)(v >> (64 - o)));
}

// Length of the match at absolute position i against i - d, up to lim - i bytes (all lanes get it).
__device__ __forceinline__ int match_len(const uint8_t* buf, int64_t i, int d, int64_t lim, int lane) {
    int len = 0;
    for (int64_t j0 = i; j0 < lim; j0 += 32) {
        const int64_t j = j0 + lane;
        const unsigned eq = __ballot_sync(0xffffffffu, j < lim && buf[j] == buf[j - d]);
        const int run = __ffs(~eq) - 1;
        if (run < 0) {
            len += 32;
            continue;
        }
        len += run;
        break;
    }
    return len;
}

__global__ void __launch_bounds__(32 * kWarps) png_deflate(Geom g) {
    __shared__ StripeSmem smem[kWarps];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t job = (int64_t)blockIdx.x * kWarps + wid;
    if (job >= (int64_t)g.n * g.stripes) return;
    StripeSmem& S = smem[wid];
    const int img = (int)(job / g.stripes), st = (int)(job % g.stripes);
    const bool last = st == g.stripes - 1;
    const uint8_t* buf = g.flt + img * g.raw;
    const int64_t s0 = (int64_t)st * g.rows * g.bpr, s1 = min(g.raw, s0 + (int64_t)g.rows * g.bpr);
    uint32_t* tok = g.tok + img * g.raw + s0;                // at most one token per byte of the stripe
    uint8_t* out = g.sbuf + job * g.stripe_cap;
    for (int s = lane; s < 286; s += 32) S.lf[s] = 0;
    if (lane < 30) S.df[lane] = 0;
    if (lane < 19) S.cf[lane] = 0;
    __syncwarp();

    // Greedy parse.  32 positions at a time, each lane tests whether its position has a candidate match of 3 or more bytes;
    // the positions before the first that has are literals.
    int64_t i = s0;
    int ntok = 0;
    while (i < s1) {
        const int64_t p = i + lane;
        bool can = false;
        if (p + 3 <= s1) {
#pragma unroll
            for (int k = 0; k < kCands; ++k) {
                const int d = g.dist[k];
                can |= d && d <= p && buf[p] == buf[p - d] && buf[p + 1] == buf[p + 1 - d] && buf[p + 2] == buf[p + 2 - d];
            }
        }
        const unsigned any = __ballot_sync(0xffffffffu, can && p < s1);
        const int q = any ? __ffs(any) - 1 : (int)min((int64_t)32, s1 - i);
        if (lane < q) {
            const uint32_t b = buf[p];
            tok[ntok + lane] = b;
            atomicAdd(&S.lf[b], 1u);
        }
        ntok += q;
        i += q;
        if (!any) continue;
        const int64_t lim = min(s1, i + kMaxMatch);
        int best = 0, bd = 0;
        for (int k = 0; k < kCands; ++k) {
            const int d = g.dist[k];
            if (!d || d > i) continue;
            const int l = match_len(buf, i, d, lim, lane);
            if (l > best) best = l, bd = d;
        }
        if (lane == 0) {
            tok[ntok] = kMatchFlag | (uint32_t)best << 16 | (uint32_t)bd;
            S.lf[257 + len_sym(best)]++;
            S.df[dist_sym(bd)]++;
        }
        ++ntok;
        i += best;
        __syncwarp();
    }
    __syncwarp();
    if (lane == 0) S.lf[256] = 1;
    __syncwarp();

    limited_lengths(S.lf, 286, 15, S.ll, S.hw);
    limited_lengths(S.df, 30, 15, S.dl, S.hw);
    int ncls = 0, hlit = 257, hdist = 1;
    if (lane == 0) {
        for (int s = 0; s < 286; ++s) if (S.ll[s]) hlit = max(hlit, s + 1);
        for (int s = 0; s < 30; ++s) if (S.dl[s]) hdist = max(hdist, s + 1);
        // run-length code of the code lengths: zeros as 18 (11-138) then 17 (3-10), other runs as the length then 16 (3-6)
        const int nl = hlit + hdist;
        auto at = [&](int k) { return k < hlit ? S.ll[k] : S.dl[k - hlit]; };
        auto emit = [&](int s, int e) { S.cls[ncls++] = (uint16_t)(s | e << 5); S.cf[s]++; };
        for (int k = 0; k < nl;) {
            const int v = at(k);
            int r = 1;
            while (k + r < nl && at(k + r) == v) ++r;
            k += r;
            if (v == 0) {
                while (r >= 11) { const int t = min(r, 138); emit(18, t - 11); r -= t; }
                if (r >= 3) { emit(17, r - 3); r = 0; }
                while (r-- > 0) emit(0, 0);
            } else {
                emit(v, 0);
                --r;
                while (r >= 3) { const int t = min(r, 6); emit(16, t - 3); r -= t; }
                while (r-- > 0) emit(v, 0);
            }
        }
    }
    ncls = __shfl_sync(0xffffffffu, ncls, 0);
    hlit = __shfl_sync(0xffffffffu, hlit, 0);
    hdist = __shfl_sync(0xffffffffu, hdist, 0);
    __syncwarp();
    limited_lengths(S.cf, 19, 7, S.cl, S.hw);
    if (lane == 0) {
        canonical_codes(S.ll, 286, S.lc);
        canonical_codes(S.dl, 30, S.dc);
        canonical_codes(S.cl, 19, S.cc);
    }
    __syncwarp();

    // size of the dynamic block
    int hclen = 4;
    for (int k = 0; k < 19; ++k) if (S.cl[c_cl_order[k]]) hclen = max(hclen, k + 1);
    int64_t bits = 0;
    for (int s = lane; s < 286; s += 32)
        bits += (int64_t)S.lf[s] * (S.ll[s] + (s >= 257 ? c_len_extra[s - 257] : 0));
    if (lane < 30) bits += (int64_t)S.df[lane] * (S.dl[lane] + c_dist_extra[lane]);
    if (lane < 19) bits += (int64_t)S.cf[lane] * (S.cl[lane] + (lane == 16 ? 2 : lane == 17 ? 3 : lane == 18 ? 7 : 0));
#pragma unroll
    for (int o = 16; o; o >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, o);
    bits += 3 + 5 + 5 + 4 + 3 * hclen;
    const int64_t dyn = last ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4;
    const int64_t raw = s1 - s0, stored = stored_bytes(raw);

    if (dyn > stored) {
        for (int64_t o = 0, c = 0; o < raw; o += kStoredMax, ++c) {
            const int k = (int)min((int64_t)kStoredMax, raw - o);
            uint8_t* h = out + o + 5 * c;
            if (lane == 0) {
                h[0] = last && o + k == raw;
                h[1] = k & 0xff, h[2] = k >> 8, h[3] = ~k & 0xff, h[4] = (~k >> 8) & 0xff;
            }
            for (int b = lane; b < k; b += 32) h[5 + b] = buf[s0 + o + b];
        }
        if (lane == 0) g.ssize[job] = stored;
        return;
    }

    unsigned long long* words = (unsigned long long*)out;
    const int nw = (int)((dyn + 7) / 8);
    for (int w = lane; w < nw; w += 32) words[w] = 0;
    __syncwarp();
    int64_t pos = 0;
    if (lane == 0) {
        auto put = [&](uint64_t v, int nb) { put_bits(words, pos, v, nb); pos += nb; };
        put((last ? 1 : 0) | 2 << 1, 3);
        put(hlit - 257, 5);
        put(hdist - 1, 5);
        put(hclen - 4, 4);
        for (int k = 0; k < hclen; ++k) put(S.cl[c_cl_order[k]], 3);
        for (int k = 0; k < ncls; ++k) {
            const int s = S.cls[k] & 31, e = S.cls[k] >> 5;
            put(S.cc[s], S.cl[s]);
            if (s >= 16) put(e, s == 16 ? 2 : s == 17 ? 3 : 7);
        }
    }
    pos = __shfl_sync(0xffffffffu, pos, 0);
    __syncwarp();
    for (int b = 0; b < ntok; b += 32) {
        int nb = 0;
        const uint64_t v = b + lane < ntok ? token_bits(tok[b + lane], S, nb) : 0;
        int incl = nb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        put_bits(words, pos + incl - nb, v, nb);
        pos += __shfl_sync(0xffffffffu, incl, 31);
    }
    __syncwarp();
    if (lane == 0) {
        put_bits(words, pos, S.lc[256], S.ll[256]);
        if (!last) {               // empty stored block after the 3 header bits (zero) and the padding: LEN 0, NLEN 0xffff
            out[dyn - 2] = 0xff;
            out[dyn - 1] = 0xff;
        }
        g.ssize[job] = dyn;
    }
}

// ------------------------------------------------------------------------------------------------------------- layout
__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = v >> 24, p[1] = v >> 16, p[2] = v >> 8, p[3] = v;
}

__device__ uint32_t crc_bytes(uint32_t c, const uint8_t* p, int n) {      // bitwise, for the short IHDR chunk
    for (int k = 0; k < n; ++k) {
        c ^= p[k];
        for (int b = 0; b < 8; ++b) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
    }
    return c;
}

constexpr uint32_t kAdlerMod = 65521;

__global__ void __launch_bounds__(256) png_layout(Geom g, uint8_t* files, int64_t* file_lens) {
    __shared__ uint64_t sa[256], sb[256];
    const int img = blockIdx.x, t = threadIdx.x;
    uint8_t* f = files + img * g.cap;
    const uint8_t* buf = g.flt + img * g.raw;
    uint64_t a = 0, b = 0;
    for (int64_t j = t; j < g.raw; j += blockDim.x) {           // Adler-32: sum x_j and sum (raw - j) x_j, mod 65521
        a += buf[j];
        b = (b + (uint64_t)((g.raw - j) % kAdlerMod) * buf[j]) % kAdlerMod;
    }
    sa[t] = a % kAdlerMod;
    sb[t] = b;
    __syncthreads();
    for (int o = blockDim.x / 2; o; o >>= 1) {
        if (t < o) sa[t] = (sa[t] + sa[t + o]) % kAdlerMod, sb[t] = (sb[t] + sb[t + o]) % kAdlerMod;
        __syncthreads();
    }
    if (t) return;
    int64_t* ss = g.ssize + (int64_t)img * g.stripes;
    int64_t off = 0;
    for (int s = 0; s < g.stripes; ++s) {
        const int64_t n = ss[s];
        ss[s] = off;
        off += n;
    }
    g.body[img] = off;
    const int64_t idat = 2 + off + 4;
    f[0] = 0x89, f[1] = 'P', f[2] = 'N', f[3] = 'G', f[4] = '\r', f[5] = '\n', f[6] = 0x1a, f[7] = '\n';
    uint8_t* ih = f + 8;
    put_be32(ih, 13);
    ih[4] = 'I', ih[5] = 'H', ih[6] = 'D', ih[7] = 'R';
    put_be32(ih + 8, g.W);
    put_be32(ih + 12, g.H);
    ih[16] = 8, ih[17] = 2, ih[18] = 0, ih[19] = 0, ih[20] = 0;
    put_be32(ih + 21, ~crc_bytes(0xffffffffu, ih + 4, 17));
    uint8_t* id = f + 33;
    put_be32(id, (uint32_t)idat);
    id[4] = 'I', id[5] = 'D', id[6] = 'A', id[7] = 'T';
    id[8] = 0x78, id[9] = 0x01;
    const uint32_t adler = (uint32_t)((sb[0] + g.raw % kAdlerMod) % kAdlerMod) << 16 | (uint32_t)((1 + sa[0]) % kAdlerMod);
    uint8_t* tail = f + kHeadBytes + off;
    put_be32(tail, adler);
    uint8_t* iend = tail + 8;
    put_be32(iend, 0);
    iend[4] = 'I', iend[5] = 'E', iend[6] = 'N', iend[7] = 'D';
    put_be32(iend + 8, 0xAE426082u);
    file_lens[img] = kHeadBytes + off + kTailBytes;
}

__global__ void __launch_bounds__(256) png_copy_stripes(Geom g, uint8_t* files) {
    const int64_t job = blockIdx.x;
    const int img = (int)(job / g.stripes), st = (int)(job % g.stripes);
    const int64_t* ss = g.ssize + (int64_t)img * g.stripes;
    const int64_t off = ss[st], end = st + 1 < g.stripes ? ss[st + 1] : g.body[img];
    const uint8_t* src = g.sbuf + job * g.stripe_cap;
    uint8_t* dst = files + img * g.cap + kHeadBytes + off;
    for (int64_t k = threadIdx.x; k < end - off; k += blockDim.x) dst[k] = src[k];
}

// ------------------------------------------------------------------------------------------------------------- CRC-32
// Reflected polynomials: bit 31 is x^0.
__device__ uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    while (true) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) return p;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
}

__device__ uint32_t x8nmodp(int64_t n) {       // x^(8n) mod P
    uint32_t r = 1u << 31, sq = 1u << 23;
    while (n) {
        if (n & 1) r = multmodp(sq, r);
        sq = multmodp(sq, sq);
        n >>= 1;
    }
    return r;
}

__device__ __forceinline__ int64_t crc_span(const Geom& g, int img) { return 4 + 2 + g.body[img] + 4; }   // "IDAT" + zlib stream

__global__ void __launch_bounds__(256) png_crc_segments(Geom g, const uint8_t* files) {
    __shared__ uint32_t table[256];
    for (int k = threadIdx.x; k < 256; k += blockDim.x) {
        uint32_t c = k;
        for (int b = 0; b < 8; ++b) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
        table[k] = c;
    }
    __syncthreads();
    const int64_t job = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (job >= (int64_t)g.n * g.nseg) return;
    const int img = (int)(job / g.nseg), seg = (int)(job % g.nseg);
    const int64_t span = crc_span(g, img), o = (int64_t)seg * kCrcSegment;
    if (o >= span) return;
    const uint8_t* p = files + img * g.cap + 37 + o;
    const int n = (int)min((int64_t)kCrcSegment, span - o);
    uint32_t c = 0;
    for (int k = 0; k < n; ++k) c = table[(c ^ p[k]) & 0xff] ^ (c >> 8);
    g.crc[job] = c;
}

__global__ void png_crc_finish(Geom g, uint8_t* files) {
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= g.n) return;
    const int64_t span = crc_span(g, img);
    const int nseg = (int)((span + kCrcSegment - 1) / kCrcSegment);
    const uint32_t full = x8nmodp(kCrcSegment);
    uint32_t c = 0xffffffffu;
    for (int s = 0; s < nseg; ++s) {
        const int64_t n = min((int64_t)kCrcSegment, span - (int64_t)s * kCrcSegment);
        c = multmodp(n == kCrcSegment ? full : x8nmodp(n), c) ^ g.crc[(int64_t)img * g.nseg + s];
    }
    put_be32(files + img * g.cap + 37 + span, ~c);
}

}  // namespace

extern "C" int n3d_png_buffer_sizes(int n, int height, int width, int64_t* scratch_bytes, int64_t* file_bytes) {
    N3D_CHECK_ARG(scratch_bytes && file_bytes, "n3d_png_buffer_sizes: null output pointer");
    Geom g;
    const int rc = make_geom(n, height, width, g);
    if (rc != N3D_OK) return rc;
    *scratch_bytes = layout(g, nullptr);
    *file_bytes = g.cap;
    return N3D_OK;
}

extern "C" int n3d_png_encode(const uint8_t* rgb, int n, int height, int width, void* scratch, uint8_t* files, int64_t* file_lens,
                              void* stream) {
    N3D_CHECK_ARG(rgb && scratch && files && file_lens, "n3d_png_encode: null buffer");
    Geom g;
    const int rc = make_geom(n, height, width, g);
    if (rc != N3D_OK) return rc;
    layout(g, (uint8_t*)scratch);
    const cudaStream_t s = (cudaStream_t)stream;
    const int64_t rows = (int64_t)n * height, jobs = (int64_t)n * g.stripes, segs = (int64_t)n * g.nseg;
    N3D_CHECK_ARG(rows <= 0x7fffffffLL * 4 / 128 && jobs < 0x7fffffffLL && segs < 0x7fffffffLL, "n3d_png_encode: batch too large");
    png_filter_rows<<<n3d_div_up(rows, 4), 128, 0, s>>>(rgb, g);
    png_deflate<<<n3d_div_up(jobs, kWarps), 32 * kWarps, 0, s>>>(g);
    png_layout<<<n, 256, 0, s>>>(g, files, file_lens);
    png_copy_stripes<<<(unsigned)jobs, 256, 0, s>>>(g, files);
    png_crc_segments<<<n3d_div_up(segs, 256), 256, 0, s>>>(g, files);
    png_crc_finish<<<n3d_div_up(n, 128), 128, 0, s>>>(g, files);
    N3D_CHECK_LAUNCH("n3d_png_encode");
    return N3D_OK;
}
