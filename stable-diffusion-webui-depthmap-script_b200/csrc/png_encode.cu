// PNG encoding of image batches on the device (include/depthmap_b200.h, "P1"): the funnel's depth, stereo and normal-map images
// leave the device as finished PNG files.
//
//   png_filter_kernel    one CTA per scanline: PNG filters 0-4, one per row by libpng's minimum-sum-of-absolute-signed-bytes
//                        rule, 16-bit samples big-endian (optionally XOR 0xFFFF), into the filtered stream [B][S]
//   png_deflate_kernel   one CTA per SEG-byte segment of an image's filtered stream: LZ77 inside the segment, its own dynamic
//                        Huffman code (or the fixed code, or a stored block, whichever is smallest), byte-aligned end
//   png_sizes_kernel     per-image file size, chunk positions, Adler-32, and the device prefix sum of the file offsets
//   png_assemble_kernel  signature, IHDR, one IDAT per segment (the first carries the zlib header), the Adler-32 IDAT, IEND;
//                        each chunk with its own CRC-32
//
// Everything a CTA computes comes from its own segment: integer histograms, prefix sums and OR-ing disjoint bits, no float
// arithmetic and no order-dependent atomics.  So an image's file is a function of that image alone (not of its batch, the call
// or the number of SMs).
#include "common.cuh"

namespace dm {
namespace png {

constexpr int SEG = 32768;                 // filtered bytes per deflate segment; also the largest match distance + 1
constexpr int SEG_CAP = SEG + 64;          // a segment's compressed bytes never exceed a stored block + sync marker (SEG + 10)
constexpr int FILTER_THREADS = 256;
constexpr int DEFLATE_THREADS = 512;
constexpr int DEFLATE_WARPS = DEFLATE_THREADS / 32;
constexpr int HASH_BITS = 12, HASH_SIZE = 1 << HASH_BITS, WAYS = 4;
constexpr int MIN_MATCH = 3, MAX_MATCH = 258;
constexpr uint32_t ADLER_MOD = 65521;
constexpr uint32_t COVERED = 1;            // info[] of a position inside an emitted match (a real match has length >= 3)
constexpr int DATA_BYTES = SEG + 512;      // the segment, zero padded so that 4-byte compares may read past its end
constexpr int UNION_BYTES = 49152;         // hash table + chunk heads, then Huffman scratch, then the output bits
constexpr size_t DEFLATE_SMEM = (size_t)SEG * 4 + DATA_BYTES + UNION_BYTES;
constexpr int ASSEMBLE_THREADS = 256;
constexpr uint32_t CRC_POLY = 0xEDB88320u;

static_assert(SEG_CAP + 64 <= UNION_BYTES, "output bits must fit the union region");
static_assert(HASH_SIZE * WAYS * 2 + HASH_SIZE * 4 <= UNION_BYTES, "hash table must fit the union region");

struct Img {
    const void *p;
    int H, W, bytes;      // bytes per sample: 2 (uint16 grey) or 1 (uint8 RGB)
    int rowbytes;         // W * C * bytes
    uint32_t inv;         // XOR applied to every 16-bit sample
};

__device__ __forceinline__ int raw_byte(const Img &im, int b, int y, int x) {
    if (im.bytes == 2) {
        const uint32_t s = reinterpret_cast<const uint16_t *>(im.p)[((size_t)b * im.H + y) * im.W + (x >> 1)] ^ im.inv;
        return (x & 1) ? (int)(s & 0xFFu) : (int)((s >> 8) & 0xFFu);
    }
    return reinterpret_cast<const uint8_t *>(im.p)[((size_t)b * im.H + y) * im.rowbytes + x];
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// |v| of the filtered byte v read as a signed char (libpng's filter heuristic)
__device__ __forceinline__ uint32_t sabs(int v) {
    const uint32_t u = (uint32_t)v & 0xFFu;
    return u < 128u ? u : 256u - u;
}

__device__ __forceinline__ int predictor(int f, int a, int u, int c) {
    switch (f) {
        case 1: return a;
        case 2: return u;
        case 3: return (a + u) >> 1;
        case 4: return paeth(a, u, c);
        default: return 0;
    }
}

__global__ void __launch_bounds__(FILTER_THREADS) png_filter_kernel(Img im, int bpp, uint8_t *filt, long long S) {
    const int y = blockIdx.x, b = blockIdx.y;
    __shared__ uint32_t red[FILTER_THREADS / 32][5];
    __shared__ int best_f;
    uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
    for (int x = threadIdx.x; x < im.rowbytes; x += FILTER_THREADS) {
        const int r = raw_byte(im, b, y, x);
        const int a = x >= bpp ? raw_byte(im, b, y, x - bpp) : 0;
        const int u = y > 0 ? raw_byte(im, b, y - 1, x) : 0;
        const int c = (x >= bpp && y > 0) ? raw_byte(im, b, y - 1, x - bpp) : 0;
        s0 += sabs(r);
        s1 += sabs(r - a);
        s2 += sabs(r - u);
        s3 += sabs(r - ((a + u) >> 1));
        s4 += sabs(r - paeth(a, u, c));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        s3 += __shfl_xor_sync(0xffffffffu, s3, o);
        s4 += __shfl_xor_sync(0xffffffffu, s4, o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        red[warp][0] = s0; red[warp][1] = s1; red[warp][2] = s2; red[warp][3] = s3; red[warp][4] = s4;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t best = 0xFFFFFFFFu;
        int bf = 0;
        for (int f = 0; f < 5; ++f) {
            uint32_t s = 0;
            for (int w = 0; w < FILTER_THREADS / 32; ++w) s += red[w][f];
            if (s < best) { best = s; bf = f; }   // ties keep the lower filter type
        }
        best_f = bf;
    }
    __syncthreads();
    const int f = best_f;
    uint8_t *row = filt + (size_t)b * S + (size_t)y * (im.rowbytes + 1);
    if (threadIdx.x == 0) row[0] = (uint8_t)f;
    for (int x = threadIdx.x; x < im.rowbytes; x += FILTER_THREADS) {
        const int r = raw_byte(im, b, y, x);
        const int a = (f == 1 || f == 3 || f == 4) && x >= bpp ? raw_byte(im, b, y, x - bpp) : 0;
        const int u = f >= 2 && y > 0 ? raw_byte(im, b, y - 1, x) : 0;
        const int c = f == 4 && x >= bpp && y > 0 ? raw_byte(im, b, y - 1, x - bpp) : 0;
        row[1 + x] = (uint8_t)(r - predictor(f, a, u, c));
    }
}

// ----------------------------------------------------------------------------------------------------------------------------
// deflate
// ----------------------------------------------------------------------------------------------------------------------------
// length symbol 257 + c for a match length 3..258, its base and extra bits (RFC 1951 3.2.5)
__device__ __forceinline__ int len_code(int len) {
    const int l = len - 3;
    if (l < 8) return l;
    if (len == 258) return 28;
    const int e = 31 - __clz(l) - 2;
    return 4 * e + 4 + ((l >> e) & 3);
}
__device__ __forceinline__ int len_extra(int c) { return (c < 8 || c == 28) ? 0 : (c - 4) >> 2; }
__device__ __forceinline__ int len_base(int c) {
    if (c < 8) return 3 + c;
    if (c == 28) return 258;
    return ((4 + (c & 3)) << ((c - 4) >> 2)) + 3;
}
// distance code for a distance 1..32768
__device__ __forceinline__ int dist_code(int dist) {
    const int d = dist - 1;
    if (d < 4) return d;
    const int e = 31 - __clz(d) - 1;
    return 2 * e + 2 + ((d >> e) & 1);
}
__device__ __forceinline__ int dist_extra(int c) { return c < 4 ? 0 : (c >> 1) - 1; }
__device__ __forceinline__ int dist_base(int c) { return c < 4 ? c + 1 : ((2 + (c & 1)) << ((c >> 1) - 1)) + 1; }

// bytes pos .. pos + 3 of the segment, little-endian
__device__ __forceinline__ uint32_t load4(const uint32_t *w, int pos) {
    const int q = pos >> 2;
    return __funnelshift_r(w[q], w[q + 1], (pos & 3) * 8);
}

__device__ __forceinline__ int match_len(const uint32_t *w, int i, int j, int maxlen) {
    int l = 0;
    while (l < maxlen) {
        const uint32_t x = load4(w, i + l) ^ load4(w, j + l);
        if (x) { l += (__ffs(x) - 1) >> 3; break; }
        l += 4;
    }
    return l < maxlen ? l : maxlen;
}

__device__ __forceinline__ uint32_t hash3(const uint32_t *w, int i) {
    return ((load4(w, i) & 0xFFFFFFu) * 2654435761u) >> (32 - HASH_BITS);
}

// OR `nbits` (<= 32) bits of v into the LSB-first bit stream at bit `pos`; the target bits are zero and no other writer owns them
__device__ __forceinline__ void put_bits(uint32_t *out, uint32_t pos, uint32_t v, int nbits) {
    if (nbits == 0) return;
    const uint32_t w = pos >> 5, sh = pos & 31;
    atomicOr(&out[w], v << sh);
    if (sh + nbits > 32) atomicOr(&out[w + 1], v >> (32 - sh));
}

// Huffman code lengths of the n symbols of `freq`, at most maxbits long, for a deflate code: complete (Kraft sum one), at least
// two codes.  sorted[0 .. nnz) = the used symbols by ascending (frequency, symbol).  One thread; `w`, `parent`, `depth` scratch of
// 2n entries.  Deterministic: a two-queue Huffman merge (ties take the leaf), then a length limit by deepening the rarest short
// codes and shortening the most frequent deepest ones.
__device__ void huffman_lengths(const uint32_t *freq, int n, int maxbits, const uint16_t *sorted, int nnz, uint8_t *lens,
                                uint32_t *w, uint16_t *parent, uint8_t *depth) {
    for (int s = 0; s < n; ++s) lens[s] = 0;
    if (nnz == 0) { lens[0] = 1; lens[1] = 1; return; }
    if (nnz == 1) { lens[sorted[0]] = 1; lens[sorted[0] == 0 ? 1 : 0] = 1; return; }
    for (int k = 0; k < nnz; ++k) w[k] = freq[sorted[k]];
    int li = 0, ii = nnz, next = nnz;
    for (int step = 0; step < nnz - 1; ++step) {
        int pick[2];
        for (int t = 0; t < 2; ++t) {
            if (li < nnz && (ii >= next || w[li] <= w[ii])) pick[t] = li++;
            else pick[t] = ii++;
        }
        w[next] = w[pick[0]] + w[pick[1]];
        parent[pick[0]] = (uint16_t)next;
        parent[pick[1]] = (uint16_t)next;
        ++next;
    }
    const int root = next - 1;
    depth[root] = 0;
    for (int v = root - 1; v >= 0; --v) depth[v] = (uint8_t)(depth[parent[v]] + 1);
    int maxlen = 0;
    for (int k = 0; k < nnz; ++k) maxlen = depth[k] > maxlen ? depth[k] : maxlen;
    for (int k = 0; k < nnz; ++k) lens[sorted[k]] = (uint8_t)(depth[k] > maxbits ? maxbits : depth[k]);
    if (maxlen <= maxbits) return;
    const uint32_t full = 1u << maxbits;
    uint32_t kraft = 0;
    for (int k = 0; k < nnz; ++k) kraft += 1u << (maxbits - lens[sorted[k]]);
    while (kraft > full) {              // deepen the rarest of the deepest codes shorter than maxbits
        int pick = -1, pl = 0;
        for (int k = 0; k < nnz; ++k) {
            const int l = lens[sorted[k]];
            if (l < maxbits && l > pl) { pl = l; pick = k; }
        }
        lens[sorted[pick]] = (uint8_t)(pl + 1);
        kraft -= 1u << (maxbits - pl - 1);
    }
    while (kraft < full) {              // shorten the most frequent of the deepest codes while the sum stays <= 1
        int pick = -1, pl = 0;
        for (int k = nnz - 1; k >= 0; --k) {
            const int l = lens[sorted[k]];
            if (l > pl) { pl = l; pick = k; }
        }
        lens[sorted[pick]] = (uint8_t)(pl - 1);
        kraft += 1u << (maxbits - pl);
    }
}

// canonical codes (RFC 1951 3.2.2), bit-reversed for the LSB-first stream
__device__ void canonical_codes(const uint8_t *lens, int n, uint16_t *codes) {
    uint16_t count[16] = {0}, next[16];
    for (int s = 0; s < n; ++s) count[lens[s]]++;
    count[0] = 0;
    uint32_t code = 0;
    for (int b = 1; b < 16; ++b) {
        code = (code + count[b - 1]) << 1;
        next[b] = (uint16_t)code;
    }
    for (int s = 0; s < n; ++s) {
        const int l = lens[s];
        codes[s] = l ? (uint16_t)(__brev((uint32_t)next[l]++) >> (32 - l)) : 0;
    }
}

__device__ __forceinline__ int fixed_lit_len(int s) { return s < 144 ? 8 : (s < 256 ? 9 : (s < 280 ? 7 : 8)); }

struct BitWriter {
    uint32_t *out;
    uint32_t pos;
    __device__ void put(uint32_t v, int n) {
        if (n == 0) return;
        const uint32_t w = pos >> 5, sh = pos & 31;
        out[w] |= v << sh;
        if (sh + n > 32) out[w + 1] |= v >> (32 - sh);
        pos += n;
    }
};

__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct SegOut {          // per (image, segment) results in the workspace
    uint32_t bytes;      // compressed bytes of the segment
    uint32_t adler_a;    // sum of the segment's bytes mod 65521
    uint32_t adler_w;    // sum of (S - global index) * byte mod 65521
    uint32_t pad;
};

// the cost in bits of the token at position p (0 inside a match)
struct Codes {
    uint8_t lit_len[288];
    uint8_t dist_len[32];
    uint16_t lit_code[288];
    uint16_t dist_code[32];
};

__device__ __forceinline__ uint32_t token_bits(const Codes &cd, uint32_t v, int byte) {
    if (v == 0) return cd.lit_len[byte];
    if (v == COVERED) return 0;
    const int lc = len_code(v & 0xFFFF), dc = dist_code((int)(v >> 16));
    return cd.lit_len[257 + lc] + len_extra(lc) + cd.dist_len[dc] + dist_extra(dc);
}

__global__ void __launch_bounds__(DEFLATE_THREADS, 1)
png_deflate_kernel(const uint8_t *filt, long long S, int nseg, int row_len, SegOut *segs, uint8_t *seg_bytes) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *info = reinterpret_cast<uint32_t *>(smem);                    // per position: 0 literal, (dist << 16 | len) match
    uint32_t *dataw = info + SEG;                                           // the segment's bytes
    uint8_t *data = reinterpret_cast<uint8_t *>(dataw);
    uint8_t *uni = data + DATA_BYTES;
    uint16_t *table = reinterpret_cast<uint16_t *>(uni);                    // phase 1: WAYS latest positions per hash
    int *chead = reinterpret_cast<int *>(uni + HASH_SIZE * WAYS * 2);       //          latest position per hash in a chunk
    uint32_t *outw = reinterpret_cast<uint32_t *>(uni);                     // phase 3: the output bits

    __shared__ uint32_t flit[288], fdist[32], fcl[19];
    __shared__ uint16_t sorted_lit[288], sorted_dist[32];
    __shared__ Codes cd;
    __shared__ uint8_t cl_len[19];
    __shared__ uint16_t cl_code[19];
    __shared__ uint16_t rle[320];
    __shared__ uint32_t warp_sum[DEFLATE_WARPS];
    __shared__ uint64_t red_a[DEFLATE_WARPS], red_w[DEFLATE_WARPS];
    __shared__ int s_mode, s_nrle, s_hlit, s_hdist, s_hclen, s_nnz_lit, s_nnz_dist;
    __shared__ uint32_t s_hdr_bits;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k = blockIdx.x, b = blockIdx.y;
    const long long seg0 = (long long)k * SEG;
    const int n = (int)(S - seg0 < SEG ? S - seg0 : SEG);
    const bool last = k == nseg - 1;
    const uint8_t *src = filt + (size_t)b * S + seg0;

    // load the segment and clear the tables; Adler-32 partial sums on the way
    uint64_t a_sum = 0, w_sum = 0;
    for (int i = tid; i < DATA_BYTES; i += DEFLATE_THREADS) {
        const uint32_t v = i < n ? src[i] : 0u;
        data[i] = (uint8_t)v;
        if (i < n) {
            a_sum += v;
            w_sum += (uint64_t)((S - seg0 - i) % ADLER_MOD) * v;
        }
    }
    for (int i = tid; i < HASH_SIZE * WAYS; i += DEFLATE_THREADS) table[i] = 0xFFFFu;
    for (int i = tid; i < HASH_SIZE; i += DEFLATE_THREADS) chead[i] = -1;
    for (int i = tid; i < 288; i += DEFLATE_THREADS) flit[i] = i == 256 ? 1u : 0u;    // one end-of-block
    if (tid < 32) fdist[tid] = 0;
    if (tid < 19) fcl[tid] = 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a_sum += __shfl_xor_sync(0xffffffffu, a_sum, o);
        w_sum += __shfl_xor_sync(0xffffffffu, w_sum, o);
    }
    if (lane == 0) { red_a[warp] = a_sum % ADLER_MOD; red_w[warp] = w_sum % ADLER_MOD; }
    __syncthreads();
    if (tid == 0) {
        uint64_t A = 0, W = 0;
        for (int i = 0; i < DEFLATE_WARPS; ++i) { A += red_a[i]; W += red_w[i]; }
        segs[(size_t)b * nseg + k].adler_a = (uint32_t)(A % ADLER_MOD);
        segs[(size_t)b * nseg + k].adler_w = (uint32_t)(W % ADLER_MOD);
    }

    // phase 1: the longest match of every position (ties: the nearest), in chunks of DEFLATE_THREADS positions.  Candidates: the
    // WAYS latest positions of earlier chunks with the same 3-byte hash, and fixed distances (runs, pixels, the row above).
    const int fixed_d[8] = {1, 2, 3, 4, 6, 8, row_len, 2 * row_len};
    for (int c0 = 0; c0 < n; c0 += DEFLATE_THREADS) {
        const int i = c0 + tid;
        const int maxlen = min(MAX_MATCH, n - i);
        const bool hv = i < n && maxlen >= MIN_MATCH;
        uint32_t h = 0;
        if (hv) {
            h = hash3(dataw, i);
            const uint32_t head = load4(dataw, i) & 0xFFFFFFu;
            int best = 0, bd = 0;
            auto consider = [&](int j) {
                const int d = i - j;
                if (j < 0 || d <= 0 || best >= maxlen) return;
                if ((load4(dataw, j) & 0xFFFFFFu) != head) return;
                if (best >= MIN_MATCH && data[j + best] != data[i + best]) return;
                const int l = match_len(dataw, i, j, maxlen);
                if (l > best || (l == best && d < bd)) { best = l; bd = d; }
            };
#pragma unroll
            for (int f = 0; f < 8; ++f) consider(i - fixed_d[f]);
            const uint16_t *t = table + h * WAYS;
#pragma unroll
            for (int wy = 0; wy < WAYS; ++wy) {
                const uint32_t j = t[wy];
                if (j != 0xFFFFu) consider((int)j);
            }
            info[i] = best >= MIN_MATCH ? ((uint32_t)bd << 16) | (uint32_t)best : 0u;
        } else if (i < n) {
            info[i] = 0;
        }
        __syncthreads();
        if (hv) atomicMax(&chead[h], i);
        __syncthreads();
        const bool win = hv && chead[h] == i;
        if (win) {
            uint16_t *t = table + h * WAYS;
#pragma unroll
            for (int wy = WAYS - 1; wy > 0; --wy) t[wy] = t[wy - 1];
            t[0] = (uint16_t)i;
        }
        __syncthreads();
        if (win) chead[h] = -1;
    }
    __syncthreads();

    // phase 2: greedy parse with one-step lazy matching, by warp 0: literal runs are skipped 32 positions at a time, a match marks
    // the positions it covers
    if (warp == 0) {
        int pos = 0;
        while (pos < n) {
            const int q = pos + lane;
            const uint32_t v = q < n ? info[q] : 0u;
            const unsigned m = __ballot_sync(0xffffffffu, v != 0u);
            if (!m) { pos += 32; continue; }
            const int first = __ffs(m) - 1, j = pos + first;
            const int L = (int)(__shfl_sync(0xffffffffu, v, first) & 0xFFFFu);
            const int Ln = j + 1 < n ? (int)(info[j + 1] & 0xFFFFu) : 0;
            __syncwarp();
            if (Ln > L) {
                if (lane == 0) info[j] = 0u;
                __syncwarp();
                pos = j + 1;
                continue;
            }
            for (int t = 1 + lane; t < L; t += 32) info[j + t] = COVERED;
            __syncwarp();
            pos = j + L;
        }
    }
    __syncthreads();

    // histograms
    for (int i = tid; i < n; i += DEFLATE_THREADS) {
        const uint32_t v = info[i];
        if (v == 0u) atomicAdd(&flit[data[i]], 1u);
        else if (v != COVERED) {
            atomicAdd(&flit[257 + len_code(v & 0xFFFF)], 1u);
            atomicAdd(&fdist[dist_code((int)(v >> 16))], 1u);
        }
    }
    __syncthreads();
    // the used symbols by ascending (frequency, symbol)
    {
        const int nl = __syncthreads_count(tid < 286 && flit[tid] != 0u);
        const int nd = __syncthreads_count(tid >= 320 && tid < 350 && fdist[tid - 320] != 0u);
        if (tid < 286 && flit[tid]) {
            const uint32_t key = (flit[tid] << 9) | tid;
            int r = 0;
            for (int s = 0; s < 286; ++s) r += flit[s] && ((flit[s] << 9) | s) < key;
            sorted_lit[r] = (uint16_t)tid;
        }
        if (tid >= 320 && tid < 350 && fdist[tid - 320]) {
            const int me = tid - 320;
            const uint32_t key = (fdist[me] << 9) | me;
            int r = 0;
            for (int s = 0; s < 30; ++s) r += fdist[s] && ((fdist[s] << 9) | s) < key;
            sorted_dist[r] = (uint16_t)me;
        }
        if (tid == 0) { s_nnz_lit = nl; s_nnz_dist = nd; }
    }
    __syncthreads();
    // phase 3: the two codes (thread 0: literal / length, thread 32: distance), scratch in the union region
    {
        uint32_t *w = reinterpret_cast<uint32_t *>(uni);
        if (tid == 0)
            huffman_lengths(flit, 286, 15, sorted_lit, s_nnz_lit, cd.lit_len, w, reinterpret_cast<uint16_t *>(w + 640),
                            reinterpret_cast<uint8_t *>(w + 960));
        if (tid == 32)
            huffman_lengths(fdist, 30, 15, sorted_dist, s_nnz_dist, cd.dist_len, w + 2048, reinterpret_cast<uint16_t *>(w + 2048 + 640),
                            reinterpret_cast<uint8_t *>(w + 2048 + 960));
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 286; s < 288; ++s) cd.lit_len[s] = 0;
        for (int s = 30; s < 32; ++s) cd.dist_len[s] = 0;
        int hlit = 286, hdist = 30;
        while (hlit > 257 && cd.lit_len[hlit - 1] == 0) --hlit;
        while (hdist > 1 && cd.dist_len[hdist - 1] == 0) --hdist;
        // run-length coded code lengths (RFC 1951 3.2.7): symbol | repeat count << 5
        int nr = 0;
        const int total = hlit + hdist;
        int i = 0;
        while (i < total) {
            const int v = i < hlit ? cd.lit_len[i] : cd.dist_len[i - hlit];
            int run = 1;
            while (i + run < total && (i + run < hlit ? cd.lit_len[i + run] : cd.dist_len[i + run - hlit]) == v) ++run;
            i += run;
            if (v == 0) {
                while (run >= 11) { const int r = run < 138 ? run : 138; rle[nr++] = (uint16_t)(18 | ((r - 11) << 5)); fcl[18]++; run -= r; }
                if (run >= 3) { rle[nr++] = (uint16_t)(17 | ((run - 3) << 5)); fcl[17]++; run = 0; }
                while (run-- > 0) { rle[nr++] = 0; fcl[0]++; }
            } else {
                rle[nr++] = (uint16_t)v; fcl[v]++; --run;
                while (run >= 3) { const int r = run < 6 ? run : 6; rle[nr++] = (uint16_t)(16 | ((r - 3) << 5)); fcl[16]++; run -= r; }
                while (run-- > 0) { rle[nr++] = (uint16_t)v; fcl[v]++; }
            }
        }
        // the code-length code (7 bits at most), its used symbols sorted by insertion
        uint16_t srt[19];
        int nnz = 0;
        for (int s = 0; s < 19; ++s) {
            if (!fcl[s]) continue;
            int p = nnz++;
            while (p > 0 && fcl[srt[p - 1]] > fcl[s]) { srt[p] = srt[p - 1]; --p; }
            srt[p] = (uint16_t)s;
        }
        uint32_t *w = reinterpret_cast<uint32_t *>(uni) + 4096;
        huffman_lengths(fcl, 19, 7, srt, nnz, cl_len, w, reinterpret_cast<uint16_t *>(w + 64), reinterpret_cast<uint8_t *>(w + 128));
        canonical_codes(cl_len, 19, cl_code);
        int hclen = 19;
        while (hclen > 4 && cl_len[kClOrder[hclen - 1]] == 0) --hclen;
        uint64_t hdr = 5 + 5 + 4 + 3 * hclen;
        for (int r = 0; r < nr; ++r) {
            const int s = rle[r] & 31;
            hdr += cl_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
        }
        // block sizes: dynamic, fixed, stored (with the sync-flush marker after all but the last segment)
        uint64_t dyn = 3 + hdr, fix = 3, extra = 0;
        for (int s = 0; s < 286; ++s) {
            dyn += (uint64_t)flit[s] * cd.lit_len[s];
            fix += (uint64_t)flit[s] * fixed_lit_len(s);
            if (s >= 257) extra += (uint64_t)flit[s] * len_extra(s - 257);
        }
        for (int s = 0; s < 30; ++s) {
            dyn += (uint64_t)fdist[s] * cd.dist_len[s];
            fix += (uint64_t)fdist[s] * 5;
            extra += (uint64_t)fdist[s] * dist_extra(s);
        }
        dyn += extra;
        fix += extra;
        auto bytes_of = [&](uint64_t bits) { return last ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4; };
        const uint64_t stored = 5 + (uint64_t)n + (last ? 0 : 5);
        int mode = 2;
        if (bytes_of(fix) < bytes_of(dyn)) mode = 1;
        if (stored < bytes_of(mode == 2 ? dyn : fix)) mode = 0;
        if (mode == 1) {
            for (int s = 0; s < 288; ++s) cd.lit_len[s] = (uint8_t)fixed_lit_len(s);
            for (int s = 0; s < 32; ++s) cd.dist_len[s] = 5;
        }
        canonical_codes(cd.lit_len, 288, cd.lit_code);
        canonical_codes(cd.dist_len, 32, cd.dist_code);
        s_mode = mode;
        s_nrle = nr;
        s_hlit = hlit;
        s_hdist = hdist;
        s_hclen = hclen;
        s_hdr_bits = (uint32_t)(3 + (mode == 2 ? hdr : 0));
    }
    __syncthreads();
    const int mode = s_mode;
    uint8_t *dst = seg_bytes + ((size_t)b * nseg + k) * SEG_CAP;
    if (mode == 0) {                    // stored block
        for (int i = tid; i < n; i += DEFLATE_THREADS) dst[5 + i] = data[i];
        if (tid == 0) {
            dst[0] = last ? 1 : 0;
            dst[1] = (uint8_t)(n & 0xFF); dst[2] = (uint8_t)(n >> 8);
            dst[3] = (uint8_t)(~n & 0xFF); dst[4] = (uint8_t)((~n >> 8) & 0xFF);
            uint32_t bytes = 5 + n;
            if (!last) {
                dst[bytes] = 0; dst[bytes + 1] = 0; dst[bytes + 2] = 0; dst[bytes + 3] = 0xFF; dst[bytes + 4] = 0xFF;
                bytes += 5;
            }
            segs[(size_t)b * nseg + k].bytes = bytes;
        }
        return;
    }
    for (int i = tid; i < SEG_CAP / 4 + 16; i += DEFLATE_THREADS) outw[i] = 0u;
    __syncthreads();
    if (tid == 0) {                     // block header (and the dynamic code description)
        BitWriter bw{outw, 0};
        bw.put((last ? 1u : 0u) | ((uint32_t)mode << 1), 3);
        if (mode == 2) {
            bw.put((uint32_t)(s_hlit - 257), 5);
            bw.put((uint32_t)(s_hdist - 1), 5);
            bw.put((uint32_t)(s_hclen - 4), 4);
            for (int i = 0; i < s_hclen; ++i) bw.put(cl_len[kClOrder[i]], 3);
            for (int r = 0; r < s_nrle; ++r) {
                const int s = rle[r] & 31, x = rle[r] >> 5;
                bw.put(cl_code[s], cl_len[s]);
                if (s == 16) bw.put((uint32_t)x, 2);
                else if (s == 17) bw.put((uint32_t)x, 3);
                else if (s == 18) bw.put((uint32_t)x, 7);
            }
        }
    }
    // bit offsets of the tokens: warp w owns positions [w * SEG / WARPS, (w + 1) * SEG / WARPS), 32 at a time
    constexpr int PER_WARP = SEG / DEFLATE_WARPS;
    const int p0 = warp * PER_WARP;
    uint32_t mine = 0;
    for (int t = 0; t < PER_WARP; t += 32) {
        const int p = p0 + t + lane;
        if (p < n) mine += token_bits(cd, info[p], data[p]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if (lane == 0) warp_sum[warp] = mine;
    __syncthreads();
    uint32_t base = s_hdr_bits, total = 0;
    for (int i = 0; i < DEFLATE_WARPS; ++i) {
        if (i < warp) base += warp_sum[i];
        total += warp_sum[i];
    }
    for (int t = 0; t < PER_WARP; t += 32) {
        const int p = p0 + t + lane;
        const uint32_t v = p < n ? info[p] : COVERED;
        const int byte = p < n ? data[p] : 0;
        const uint32_t c = p < n ? token_bits(cd, v, byte) : 0u;
        uint32_t incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        const uint32_t at = base + incl - c;
        if (v == 0u) {
            put_bits(outw, at, cd.lit_code[byte], cd.lit_len[byte]);
        } else if (v != COVERED) {
            const int L = (int)(v & 0xFFFF), d = (int)(v >> 16);
            const int lc = len_code(L), dc = dist_code(d);
            const int ln = cd.lit_len[257 + lc], dn = cd.dist_len[dc];
            put_bits(outw, at, cd.lit_code[257 + lc] | ((uint32_t)(L - len_base(lc)) << ln), ln + len_extra(lc));
            put_bits(outw, at + ln + len_extra(lc), cd.dist_code[dc] | ((uint32_t)(d - dist_base(dc)) << dn), dn + dist_extra(dc));
        }
        base += __shfl_sync(0xffffffffu, incl, 31);
    }
    __syncthreads();
    uint32_t end_bits = s_hdr_bits + total + cd.lit_len[256];
    const uint32_t bytes = last ? (end_bits + 7) / 8 : (end_bits + 3 + 7) / 8 + 4;
    if (tid == 0) {
        put_bits(outw, s_hdr_bits + total, cd.lit_code[256], cd.lit_len[256]);
        segs[(size_t)b * nseg + k].bytes = bytes;
    }
    __syncthreads();
    const uint8_t *ob = reinterpret_cast<const uint8_t *>(outw);
    for (uint32_t i = tid; i < bytes; i += DEFLATE_THREADS) {
        uint8_t v = ob[i];
        if (!last && i + 2 >= bytes) v = 0xFF;               // the sync-flush marker 00 00 FF FF after an empty stored block
        else if (!last && i + 4 >= bytes) v = 0;
        dst[i] = v;
    }
}

// ----------------------------------------------------------------------------------------------------------------------------
// container
// ----------------------------------------------------------------------------------------------------------------------------
constexpr int FIXED_BYTES = 8 + 25 + 2 + 16 + 12;    // signature, IHDR, zlib header, Adler-32 IDAT, IEND

__global__ void png_sizes_kernel(const SegOut *segs, int B, int nseg, long long S, uint64_t *chunk_pos, uint32_t *adler,
                                 int64_t *offsets) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        uint64_t pos = 33, A = 1, W = (uint64_t)(S % ADLER_MOD);
        for (int k = 0; k < nseg; ++k) {
            const SegOut s = segs[(size_t)b * nseg + k];
            chunk_pos[(size_t)b * nseg + k] = pos;
            pos += 12 + s.bytes + (k == 0 ? 2 : 0);
            A += s.adler_a;
            W += s.adler_w;
        }
        adler[b] = (uint32_t)(((W % ADLER_MOD) << 16) | (A % ADLER_MOD));
        offsets[b + 1] = (int64_t)(pos + 16 + 12);          // this image's file size, summed below
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t o = 0;
        offsets[0] = 0;
        for (int b = 0; b < B; ++b) { o += offsets[b + 1]; offsets[b + 1] = o; }
    }
}

__device__ uint32_t multmodp(uint32_t a, uint32_t b) {      // a * b modulo the CRC-32 polynomial (reflected), a != 0
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}

__device__ uint32_t x8nmodp(uint64_t n) {                   // x^(8n) modulo the polynomial
    uint32_t p = 1u << 31, sq = 1u << 23;                   // x^0, x^8
    while (n) {
        if (n & 1) p = multmodp(sq, p);
        sq = multmodp(sq, sq);
        n >>= 1;
    }
    return p;
}

__device__ __forceinline__ void put_be32(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

__device__ uint32_t crc_serial(const uint32_t *tab, const uint8_t *p, int n) {
    uint32_t c = 0xFFFFFFFFu;
    for (int i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
    return ~c;
}

__global__ void __launch_bounds__(ASSEMBLE_THREADS)
png_assemble_kernel(const SegOut *segs, const uint8_t *seg_bytes, const uint64_t *chunk_pos, const uint32_t *adler,
                    const int64_t *offsets, int nseg, int H, int W, int color_type, int bit_depth, uint8_t *out) {
    __shared__ uint32_t tab[256];
    __shared__ uint32_t crc[ASSEMBLE_THREADS];
    __shared__ uint32_t mult[8];
    __shared__ __align__(16) uint8_t buf[6 + SEG_CAP];
    const int tid = threadIdx.x, k = blockIdx.x, b = blockIdx.y;
    {
        uint32_t c = (uint32_t)tid;
        for (int i = 0; i < 8; ++i) c = (c & 1) ? CRC_POLY ^ (c >> 1) : c >> 1;
        tab[tid] = c;
    }
    uint8_t *file = out + offsets[b];
    __syncthreads();
    if (k == nseg) {                    // signature, IHDR, the Adler-32 IDAT, IEND
        if (tid == 0) {
            const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
            for (int i = 0; i < 8; ++i) file[i] = sig[i];
            uint8_t ih[17] = {'I', 'H', 'D', 'R'};
            put_be32(ih + 4, (uint32_t)W);
            put_be32(ih + 8, (uint32_t)H);
            ih[12] = (uint8_t)bit_depth; ih[13] = (uint8_t)color_type; ih[14] = 0; ih[15] = 0; ih[16] = 0;
            put_be32(file + 8, 13);
            for (int i = 0; i < 17; ++i) file[12 + i] = ih[i];
            put_be32(file + 29, crc_serial(tab, ih, 17));
            uint8_t *end = out + offsets[b + 1];
            uint8_t ad[8] = {'I', 'D', 'A', 'T'};
            put_be32(ad + 4, adler[b]);
            put_be32(end - 28, 4);
            for (int i = 0; i < 8; ++i) end[-24 + i] = ad[i];
            put_be32(end - 16, crc_serial(tab, ad, 8));
            const uint8_t ie[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
            for (int i = 0; i < 12; ++i) end[-12 + i] = ie[i];
        }
        return;
    }
    // IDAT k: type, (zlib header,) segment bytes; CRC-32 by 256 right-aligned pieces combined pairwise
    const int hdr = k == 0 ? 2 : 0;
    const int len = (int)segs[(size_t)b * nseg + k].bytes + hdr;
    const int n = 4 + len;
    const uint8_t *src = seg_bytes + ((size_t)b * nseg + k) * SEG_CAP;
    if (tid < 4) buf[tid] = "IDAT"[tid];
    if (tid == 0 && hdr) { buf[4] = 0x78; buf[5] = 0x5E; }
    for (int i = tid; i < len - hdr; i += ASSEMBLE_THREADS) buf[4 + hdr + i] = src[i];
    const int L = (n + ASSEMBLE_THREADS - 1) / ASSEMBLE_THREADS;
    if (tid == 0) {
        uint32_t m = x8nmodp((uint64_t)L);
        for (int s = 0; s < 8; ++s) { mult[s] = m; m = multmodp(m, m); }
    }
    __syncthreads();
    {
        const int hi = n - (ASSEMBLE_THREADS - 1 - tid) * L, lo = hi - L;
        uint32_t c = 0xFFFFFFFFu;
        for (int i = lo < 0 ? 0 : lo; i < hi; ++i) c = tab[(c ^ buf[i]) & 0xFFu] ^ (c >> 8);
        crc[tid] = hi > 0 ? ~c : 0u;
    }
    __syncthreads();
    for (int s = 0; s < 8; ++s) {
        const int stride = 1 << s;
        if ((tid & (2 * stride - 1)) == 0) crc[tid] = multmodp(mult[s], crc[tid]) ^ crc[tid + stride];
        __syncthreads();
    }
    uint8_t *chunk = file + chunk_pos[(size_t)b * nseg + k];
    if (tid == 0) {
        put_be32(chunk, (uint32_t)len);
        put_be32(chunk + 8 + len, crc[0]);
    }
    for (int i = tid; i < n; i += ASSEMBLE_THREADS) chunk[4 + i] = buf[i];
}

// OUTPUT_DEPTH_COMBINE: the RGB image and the depth's high byte on all three channels (convert_i16_to_rgb), side by side
// (horizontal) or stacked
__global__ void depth_combine_rgb_kernel(const uint8_t *rgb, const uint16_t *depth, int B, int H, int W, int horizontal, uint32_t inv,
                                         uint8_t *out) {
    const int OW = horizontal ? 2 * W : W, OH = horizontal ? H : 2 * H;
    const long long total = (long long)B * OH * OW;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(p % OW);
        const long long r = p / OW;
        const int y = (int)(r % OH), b = (int)(r / OH);
        const bool second = horizontal ? x >= W : y >= H;
        const int sx = horizontal && second ? x - W : x, sy = !horizontal && second ? y - H : y;
        const size_t s = ((size_t)b * H + sy) * W + sx;
        uint8_t *o = out + p * 3;
        if (second) {
            const uint8_t v = (uint8_t)(((uint32_t)depth[s] ^ inv) >> 8);
            o[0] = v; o[1] = v; o[2] = v;
        } else {
            o[0] = rgb[s * 3]; o[1] = rgb[s * 3 + 1]; o[2] = rgb[s * 3 + 2];
        }
    }
}

struct Layout {
    long long S;        // filtered bytes per image
    int nseg, rowbytes;
};

static bool layout_of(int H, int W, int C, int bit_depth, Layout &l) {
    if (H <= 0 || W <= 0 || !((C == 1 && bit_depth == 16) || (C == 3 && bit_depth == 8))) return false;
    const long long rb = (long long)W * C * (bit_depth / 8);
    if (rb >= (1ll << 30)) return false;
    l.rowbytes = (int)rb;
    l.S = (long long)H * (rb + 1);
    l.nseg = (int)((l.S + SEG - 1) / SEG);
    return l.S < (1ll << 40);
}

struct Ws {
    uint8_t *filt, *seg_bytes;
    SegOut *segs;
    uint64_t *chunk_pos;
    uint32_t *adler;
    size_t total;
};

static Ws carve(void *base, int B, const Layout &l) {
    Ws w;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes, 256); return at; };
    const size_t f = take((size_t)B * l.S), sb = take((size_t)B * l.nseg * SEG_CAP), sg = take((size_t)B * l.nseg * sizeof(SegOut)),
                 cp = take((size_t)B * l.nseg * sizeof(uint64_t)), ad = take((size_t)B * sizeof(uint32_t));
    uint8_t *p = static_cast<uint8_t *>(base);
    w.filt = p + f;
    w.seg_bytes = p + sb;
    w.segs = reinterpret_cast<SegOut *>(p + sg);
    w.chunk_pos = reinterpret_cast<uint64_t *>(p + cp);
    w.adler = reinterpret_cast<uint32_t *>(p + ad);
    w.total = o + 256;
    return w;
}

}  // namespace png
}  // namespace dm

extern "C" __attribute__((visibility("default"))) size_t dm_png_encode_bound(int H, int W, int C, int bit_depth) {
    dm::png::Layout l;
    if (!dm::png::layout_of(H, W, C, bit_depth, l)) return 0;
    return (size_t)dm::png::FIXED_BYTES + (size_t)l.S + (size_t)l.nseg * 22;
}

extern "C" __attribute__((visibility("default"))) size_t dm_png_encode_workspace_bytes(int B, int H, int W, int C, int bit_depth) {
    dm::png::Layout l;
    if (B <= 0 || !dm::png::layout_of(H, W, C, bit_depth, l)) return 0;
    return dm::png::carve(nullptr, B, l).total;
}

extern "C" __attribute__((visibility("default"))) int dm_png_encode(const void *img, int B, int H, int W, int C, int bit_depth, int flags,
                                                                 uint8_t *out, size_t out_capacity, int64_t *offsets, void *workspace,
                                                                 size_t workspace_bytes, void *stream_) {
    using namespace dm;
    using namespace dm::png;
    Layout l;
    if (!img || !out || !offsets || B <= 0 || B > 65535 || !layout_of(H, W, C, bit_depth, l) || (flags & ~DM_PNG_INVERT) ||
        ((flags & DM_PNG_INVERT) && bit_depth != 16)) {
        set_error("dm_png_encode: bad arguments (uint16 [B,H,W] with C = 1, bit_depth 16, or uint8 [B,H,W,3] with C = 3, bit_depth 8; "
                  "DM_PNG_INVERT only on 16-bit images)");
        return DM_E_INVALID;
    }
    const size_t bound = dm_png_encode_bound(H, W, C, bit_depth);
    if (out_capacity / (size_t)B < bound) {
        set_error("dm_png_encode: output capacity %zu is below B * dm_png_encode_bound = %zu", out_capacity, bound * (size_t)B);
        return DM_E_WORKSPACE;
    }
    const size_t need = dm_png_encode_workspace_bytes(B, H, W, C, bit_depth);
    if (!workspace || workspace_bytes < need) {
        set_error("dm_png_encode: workspace of %zu bytes is below the %zu of dm_png_encode_workspace_bytes", workspace_bytes, need);
        return DM_E_WORKSPACE;
    }
    cudaStream_t stream = (cudaStream_t)stream_;
    static PerDeviceFlag configured;
    if (!configured.test_and_set())
        DM_CUDA_CHECK(cudaFuncSetAttribute(png_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DEFLATE_SMEM));
    const Ws ws = carve(workspace, B, l);
    const Img im{img, H, W, bit_depth / 8, l.rowbytes, (flags & DM_PNG_INVERT) ? 0xFFFFu : 0u};
    png_filter_kernel<<<dim3((unsigned)H, (unsigned)B), FILTER_THREADS, 0, stream>>>(im, C * (bit_depth / 8), ws.filt, l.S);
    DM_LAUNCH_CHECK("png_filter_kernel");
    png_deflate_kernel<<<dim3((unsigned)l.nseg, (unsigned)B), DEFLATE_THREADS, DEFLATE_SMEM, stream>>>(
        ws.filt, l.S, l.nseg, l.rowbytes + 1, ws.segs, ws.seg_bytes);
    DM_LAUNCH_CHECK("png_deflate_kernel");
    png_sizes_kernel<<<1, 256, 0, stream>>>(ws.segs, B, l.nseg, l.S, ws.chunk_pos, ws.adler, offsets);
    DM_LAUNCH_CHECK("png_sizes_kernel");
    png_assemble_kernel<<<dim3((unsigned)l.nseg + 1, (unsigned)B), ASSEMBLE_THREADS, 0, stream>>>(
        ws.segs, ws.seg_bytes, ws.chunk_pos, ws.adler, offsets, l.nseg, H, W, C == 1 ? 0 : 2, bit_depth, out);
    DM_LAUNCH_CHECK("png_assemble_kernel");
    return DM_OK;
}

extern "C" __attribute__((visibility("default"))) int dm_depth_combine_rgb(const uint8_t *rgb, const uint16_t *depth, int B, int H, int W,
                                                                        int horizontal, int invert, uint8_t *out, void *stream_) {
    using namespace dm;
    if (!rgb || !depth || !out || B <= 0 || H <= 0 || W <= 0) { set_error("dm_depth_combine_rgb: bad arguments"); return DM_E_INVALID; }
    const long long total = (long long)B * H * W * 2;
    const int T = 256;
    const unsigned grid = (unsigned)((total + T - 1) / T < 65536 * 16 ? (total + T - 1) / T : 65536 * 16);
    png::depth_combine_rgb_kernel<<<grid, T, 0, (cudaStream_t)stream_>>>(rgb, depth, B, H, W, horizontal ? 1 : 0, invert ? 0xFFFFu : 0u, out);
    DM_LAUNCH_CHECK("depth_combine_rgb_kernel");
    return DM_OK;
}
