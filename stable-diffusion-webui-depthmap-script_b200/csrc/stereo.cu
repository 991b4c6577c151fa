// S1-S5 — stereo pair generation.  Replaces src/stereoimage_generation.py:13-307 of the reference.
//
// One CTA owns one image row (rows are independent in every fill mode, :101/:174) and produces BOTH eyes for it from
// a single read of the row (3 B/px RGB + 2 B/px depth), writing the packed result once (6 B/px SBS, 3 B/px anaglyph):
// the compulsory 11 B/px (8 B/px anaglyph) of SURVEY §8d and nothing else touches HBM.
//
// The reference's row algorithms are sequential sweeps; they are re-derived here as data-parallel forms that give the
// same bytes (compiled with -fmad=false: numba emits no FMA contraction; all arithmetic fp64 like the reference):
//
//  naive family (:95-159)  forward scatter where "the last writer in sweep order wins" == atomicMax (div_px < 0,
//      ascending sweep) / atomicMin (otherwise) of the SOURCE column per destination.  `naive` fill = nearest filled
//      neighbour, right before left, within |int(div_px)|+1.  `naive_interpolating` = closed form of the left-to-right
//      gap walk: with V = filled & non-black, a pixel p lies in a gap iff an unfilled pixel exists in (lastV(p), p];
//      the gap is [first such pixel, next V after p) and its borders are read from the pre-fill row (three scans).
//
//  polylines (:162-283)  the morphed polyline never self-intersects (proof in the reference, :200-212), so at any x
//      the segment with maximal closeness is the FIRST (div_px >= 0) or LAST (div_px < 0) segment, in original vertex
//      order, that spans x.  Hence winner(x) = (first t with prefixmax(X)[t] >= x) - 1, resp. last t with
//      suffixmin(X)[t] < x: one scan + one binary search replaces the active-segment list.  The stable insertion sort
//      becomes a counting sort by floor(x) (one bucket per output pixel) + an in-bucket insertion sort on (x, index).
//      Each output pixel then walks its own sub-intervals in sorted order, accumulating colour*significance from 0.5
//      exactly as :229-281 does, and truncates.  Distinct non-adjacent spanning segments differ in closeness by >= 0.1
//      (sharp) / 1 (soft) px, 12 orders of magnitude above fp64 rounding, so the reformulation is exact except on
//      exact ties of vertex x (measure-zero; stable order is still honoured for the sub-interval sequence).
#include <math.h>

#include "common.cuh"

namespace dm {

struct StereoArgs {
    const uint8_t *rgb;
    const void *depth;
    const uint32_t *minmax;  // [B][2] u16 min / max (DM_DEPTH_U16 only)
    int H, W;
    double exponent;
    double div_px[2], sep_px[2];
    int eye_mode[2];
    int fill, pack, red_eye, depth_kind;
    double *dbg;    // debug dump (tests only): row 0 / image 0 / first warped eye -> [n, pm[n], order[n], off[W+2]]
    uint8_t *out[2];
    int64_t row_stride[2], img_stride[2];
};

constexpr double EPSILON = 1e-7;

// ---------------------------------------------------------------------------------------------------------------
// block-wide inclusive scans over shared memory (chunk per thread + shuffle scan of chunk totals)
// ---------------------------------------------------------------------------------------------------------------
template <typename T, typename Op>
__device__ void block_scan_inclusive(T *data, int n, T identity, Op op, bool reverse, T *warp_tot /*[32]*/) {
    const int T_ = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int chunk = (n + T_ - 1) / T_;
    const int beg = tid * chunk, end = min(n, beg + chunk);
    T acc = identity;
    for (int i = beg; i < end; ++i) {
        const int j = reverse ? n - 1 - i : i;
        acc = op(acc, data[j]);
        data[j] = acc;
    }
    // exclusive scan of per-thread totals
    T incl = acc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        T v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl = op(v, incl);
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        T w = lane < (T_ >> 5) ? warp_tot[lane] : identity;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            T v = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w = op(v, w);
        }
        warp_tot[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    T excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = identity;
    if (warp > 0) excl = op(warp_tot[warp - 1], excl);
    for (int i = beg; i < end; ++i) {
        const int j = reverse ? n - 1 - i : i;
        data[j] = op(excl, data[j]);
    }
    __syncthreads();
}

struct OpMaxD { __device__ double operator()(double a, double b) const { return b > a ? b : a; } };
struct OpMinD { __device__ double operator()(double a, double b) const { return b < a ? b : a; } };
struct OpMaxI { __device__ int operator()(int a, int b) const { return max(a, b); } };
struct OpMinI { __device__ int operator()(int a, int b) const { return min(a, b); } };
struct OpAddI { __device__ int operator()(int a, int b) const { return a + b; } };

// coalesced store of `nbytes` from shared `src` to global `dst` (arbitrary alignment)
__device__ __forceinline__ void store_row(uint8_t *dst, const uint8_t *src, int nbytes) {
    const int tid = threadIdx.x, T_ = blockDim.x;
    const int head = (int)((16 - ((uintptr_t)dst & 15)) & 15);
    const int h = head < nbytes ? head : nbytes;
    for (int i = tid; i < h; i += T_) dst[i] = src[i];
    const int nvec = (nbytes - h) >> 4;
    for (int i = tid; i < nvec; i += T_) {
        const uint8_t *s = src + h + i * 16;
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
            w[k] = (uint32_t)s[4 * k] | ((uint32_t)s[4 * k + 1] << 8) | ((uint32_t)s[4 * k + 2] << 16) | ((uint32_t)s[4 * k + 3] << 24);
        *reinterpret_cast<uint4 *>(dst + h + i * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    const int tail0 = h + nvec * 16;
    for (int i = tail0 + tid; i < nbytes; i += T_) dst[i] = src[i];
}

__device__ __forceinline__ double pow_ref(double nd, double e, int kind) {
    // kind 0: e == 1 (pow(x,1) == x exactly); 1: e == 2 (x*x, correctly rounded); 2: general (CUDA pow, <= 2 ulp)
    if (kind == 0) return nd;
    if (kind == 1) return nd * nd;
    return pow(nd, e);
}

__device__ __forceinline__ uint8_t f64_to_u8_wrap(double v) {
    if (!(v > -2.0e9 && v < 2.0e9)) return 0;
    return (uint8_t)(int)v;
}

// ---------------------------------------------------------------------------------------------------------------
// the row kernel
// ---------------------------------------------------------------------------------------------------------------
// All row state lives in dynamic shared memory.  The carve-up is kept as BYTE OFFSETS from the file-scope `g_smem`
// symbol (not as generic pointers inside a struct) so the compiler keeps the shared address space and emits LDS / STS
// instead of generic LD / ST (the first version's ncu source page showed LD.E / ST.E on every row access).
extern __shared__ __align__(16) uint8_t g_smem[];

struct RowSmem {
    uint32_t src;      // u8  [3W] (naive family)  |  u32 [W] R | G<<8 | B<<16 (polylines)
    uint32_t eye[2];   // u8  [3W] each
    uint32_t ndp;      // f64 [W]   nd ** exponent
    uint32_t xs;       // f64 [n]   vertex x in original order (polylines)
    uint32_t pm;       // f64 [n]   prefix max / suffix min of vertex x (polylines); u8 [3W] scatter staging (naive)
    uint32_t order;    // u16 [n]   vertex indices sorted by (x, index) (polylines)
    uint32_t off;      // i32 [W+3] bucket offsets (polylines) / winner + filled (naive)
    uint32_t cur;      // i32 [W+3] bucket cursors (polylines) / lastV (naive_interpolating)
    uint32_t aux;      // i32 [W+1] nextV (naive_interpolating)
    uint32_t wtot_d;   // f64 [32]
    uint32_t wtot_i;   // i32 [32]
    template <typename T>
    __device__ __forceinline__ T *at(uint32_t o) const { return reinterpret_cast<T *>(g_smem + o); }
};

// nd ** exponent of a source column: read from the fp64 row (DM_DEPTH_ND64) or recomputed from the u16 depth row kept in
// shared memory (DM_DEPTH_U16; one IEEE division, :81) — the latter saves 8 B/px of shared memory, which is what lets two
// row-CTAs share an SM at 2048 px.
struct NdSrc {
    const double *ndp;
    const uint16_t *dep;
    uint32_t mn;
    double den, rden, expo;     // rden = 1 / den, correctly rounded
    int pow_kind;
    __device__ __forceinline__ double get(int col) const {
        if (ndp) return ndp[col];
        // (d - min) / (max - min) as the reference's float64 true-divide (:81), without the division: with r = RN(1/den),
        // q0 = RN(a r), the residual a - q0 den is exact in one FMA and RN(q0 + residual r) is the correctly rounded quotient
        // (Markstein); checked for EVERY pair 0 <= a <= den <= 65535 on the CPU (tests/test_exact_division.py).
        const double a = (double)((uint32_t)dep[col] - mn);
        const double q0 = __dmul_rn(a, rden);
        const double rem = __fma_rn(-q0, den, a);
        return pow_ref(__fma_rn(rem, rden, q0), expo, pow_kind);
    }
};

__device__ __forceinline__ int vertex_bucket(double x, int W) { return x < 0.0 ? 0 : (x >= (double)W ? W + 1 : (int)x + 1); }

template <bool SHARP>
__device__ void polylines_eye(const RowSmem &sm, const NdSrc &nds, int W, double div_px, double sep_px, uint32_t dst_off, double *dbg) {
    const int tid = threadIdx.x, T_ = blockDim.x;
    const int n = SHARP ? 2 * W + 2 : W + 2;
    const bool fwd = !(div_px < 0.0);
    double *xs = sm.at<double>(sm.xs), *pm = sm.at<double>(sm.pm);
    uint16_t *order = sm.at<uint16_t>(sm.order);
    uint16_t *rk = sm.at<uint16_t>(sm.pm);          // rank inside the bucket; lives in pm's memory until pm is built
    int *off = sm.at<int>(sm.off);
    const uint32_t *src = sm.at<uint32_t>(sm.src);
    uint8_t *dst = sm.at<uint8_t>(dst_off);

    // 1. vertex x (:177-192), one source pixel per thread iteration: both vertices of a sharp pixel share nd ** e * div_px.
    //    The counting sort's histogram is taken on the way: atomicAdd returns the vertex's rank inside its bucket.
    for (int b = tid; b < W + 3; b += T_) off[b] = 0;
    __syncthreads();
    for (int col = tid; col < W; col += T_) {
        const double coord_d = nds.get(col) * div_px;
        const double coord_x = (double)col + 0.5 + coord_d + sep_px;
        if (SHARP) {
            const double xa = coord_x - 0.45, xb = coord_x + 0.45;
            xs[1 + 2 * col] = xa; xs[2 + 2 * col] = xb;
            rk[1 + 2 * col] = (uint16_t)atomicAdd(&off[vertex_bucket(xa, W)], 1);
            rk[2 + 2 * col] = (uint16_t)atomicAdd(&off[vertex_bucket(xb, W)], 1);
        } else {
            xs[1 + col] = coord_x;
            rk[1 + col] = (uint16_t)atomicAdd(&off[vertex_bucket(coord_x, W)], 1);
        }
    }
    if (tid == 0) {
        xs[0] = -1.0 * (double)W; xs[n - 1] = 2.0 * (double)W;       // sentinels; the closing one never moves (:214)
        rk[0] = (uint16_t)atomicAdd(&off[0], 1);
    }
    __syncthreads();
    // 2. bucket ends (inclusive scan): afterwards off[b] = END of bucket b = START of bucket b + 1
    block_scan_inclusive<int>(off, W + 2, 0, OpAddI(), false, sm.at<int>(sm.wtot_i));
    for (int t = tid; t < n - 1; t += T_) {
        const int b = vertex_bucket(xs[t], W);
        order[(b ? off[b - 1] : 0) + (int)rk[t]] = (uint16_t)t;
    }
    if (tid == 0) order[n - 1] = (uint16_t)(n - 1);
    __syncthreads();
    // 3. prefix max / suffix min of x in ORIGINAL order (the rank array is dead now) and the order inside buckets by (x, index)
    for (int t = tid; t < n; t += T_) pm[t] = xs[t];
    __syncthreads();
    if (fwd) block_scan_inclusive<double>(pm, n, -INFINITY, OpMaxD(), false, sm.at<double>(sm.wtot_d));
    else block_scan_inclusive<double>(pm, n, INFINITY, OpMinD(), true, sm.at<double>(sm.wtot_d));
    for (int b = tid; b < W + 2; b += T_) {
        const int beg = b ? off[b - 1] : 0, end = off[b];
        if (end - beg < 2) continue;
        if (b == 0 || b == W + 1) {
            // bucket 0: only its maximum matters (predecessor of pixel 0) -> move it last;
            // bucket W+1: only its minimum matters (successor of the last in-range vertex) -> move it first
            const bool want_max = b == 0;
            int bi = beg, bt = order[beg];
            double bx = xs[bt];
            for (int i = beg + 1; i < end; ++i) {
                const int t = order[i];
                const double x = xs[t];
                const bool better = want_max ? (x > bx || (x == bx && t > bt)) : (x < bx || (x == bx && t < bt));
                if (better) { bx = x; bt = t; bi = i; }
            }
            const int slot = want_max ? end - 1 : beg;
            const uint16_t tmp = order[slot]; order[slot] = order[bi]; order[bi] = tmp;
        } else {
            for (int i = beg + 1; i < end; ++i) {
                const int t = order[i];
                const double x = xs[t];
                int j = i - 1;
                while (j >= beg) {
                    const int tj = order[j];
                    const double xj = xs[tj];
                    if (xj > x || (xj == x && tj > t)) { order[j + 1] = (uint16_t)tj; --j; } else break;
                }
                order[j + 1] = (uint16_t)t;
            }
        }
    }
    __syncthreads();
    if (dbg && tid == 0) {
        dbg[0] = n;
        for (int t = 0; t < n; ++t) { dbg[1 + t] = pm[t]; dbg[1 + n + t] = order[t]; dbg[1 + 2 * n + t] = xs[t]; }
        for (int b = 0; b < W + 2; ++b) dbg[1 + 3 * n + b] = off[b];
    }
    // 4. rasterise: one output pixel per thread iteration (:228-281)
    for (int col = tid; col < W; col += T_) {
        double c0 = 0.5, c1 = 0.5, c2 = 0.5;
        int i = off[col] - 1;  // last vertex with x < col  (end of bucket col == number of vertices with x < col)
        int ti = order[i];
        double xi = xs[ti];
        const double colf = (double)col, colp = (double)(col + 1);
        while (xi < colp) {
            const int tn = order[i + 1];
            const double xn = xs[tn];
            const double coord_from = (xi > colf ? xi : colf) + EPSILON;
            const double coord_to = (xn < colp ? xn : colp) - EPSILON;
            const double significance = coord_to - coord_from;
            const double coord_center = coord_from + 0.5 * significance;
            // Winning segment s = vertices (s, s+1) in original order.  The left vertex of this sub-interval, ti, is the
            // natural candidate (exact wherever nothing occludes it); verify against the monotone pm[] and gallop.
            int s;
            if (fwd) {   // s + 1 = first t with pm[t] >= center
                int lo, hi;  // invariant: pm[lo] < center <= pm[hi]  (lo may be -1 conceptually: pm[0] = -W < center)
                if (pm[ti] >= coord_center) {
                    hi = ti; lo = ti - 1;
                    int step = 1;
                    while (lo > 0 && pm[lo] >= coord_center) { hi = lo; lo -= step; step <<= 1; }
                    if (lo < 0) lo = 0;
                } else {
                    lo = ti; hi = ti + 1;
                    int step = 1;
                    while (pm[hi] < coord_center) { lo = hi; hi += step; step <<= 1; if (hi > n - 1) hi = n - 1; }
                }
                while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pm[mid] >= coord_center) hi = mid; else lo = mid; }
                s = hi - 1;
            } else {     // s = last t with pm[t] < center; pm[ti] <= x_i < center always holds
                int lo = ti, hi = ti + 1, step = 1;
                while (hi < n - 1 && pm[hi] < coord_center) { lo = hi; hi += step; step <<= 1; if (hi > n - 1) hi = n - 1; }
                if (pm[hi] < coord_center) lo = hi;   // cannot happen (pm[n-1] = 2W), kept for safety
                else while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pm[mid] < coord_center) lo = mid; else hi = mid; }
                s = lo;
            }
            // Source columns of vertices s and s+1.  Written as plain clamps of the column index on purpose: with
            // CUDA 12.9 ptxas (seen on a Blackwell target; not re-examined on sm_90a), `s = min(s, n-2)` followed by a test `s == n-2` is fused into a VIMNMX with a
            // predicate output whose sense is wrong on the hardware (observed: the equality came out true for every
            // s < n-2), so no equality test may follow a min/max on the same operands here.
            int col_l = SHARP ? ((s - 1) >> 1) : (s - 1);   // vertex 0 (opening sentinel) -> -1 -> column 0
            int col_r = SHARP ? (s >> 1) : s;               // vertex n-1 (closing sentinel) -> W -> column W-1
            col_l = col_l < 0 ? 0 : (col_l > W - 1 ? W - 1 : col_l);
            col_r = col_r < 0 ? 0 : (col_r > W - 1 ? W - 1 : col_r);
            const uint32_t pl = src[col_l];
            if (col_l == col_r) {
                c0 += (double)(pl & 0xffu) * significance;
                c1 += (double)((pl >> 8) & 0xffu) * significance;
                c2 += (double)((pl >> 16) & 0xffu) * significance;
            } else {
                const uint32_t pr = src[col_r];
                const double x0 = xs[s], x1 = xs[s + 1];
                const double ip_k = (coord_center - x0) / (x1 - x0);
                const double om = 1.0 - ip_k;
                c0 += ((double)(pl & 0xffu) * om + (double)(pr & 0xffu) * ip_k) * significance;
                c1 += ((double)((pl >> 8) & 0xffu) * om + (double)((pr >> 8) & 0xffu) * ip_k) * significance;
                c2 += ((double)((pl >> 16) & 0xffu) * om + (double)((pr >> 16) & 0xffu) * ip_k) * significance;
            }
            ++i;
            ti = tn;
            xi = xn;
        }
        dst[3 * col + 0] = f64_to_u8_wrap(c0);
        dst[3 * col + 1] = f64_to_u8_wrap(c1);
        dst[3 * col + 2] = f64_to_u8_wrap(c2);
    }
    __syncthreads();
}

__device__ void naive_eye(const RowSmem &sm, const NdSrc &nds, int W, double div_px, double sep_px, int fill, uint32_t dst_off) {
    const int tid = threadIdx.x, T_ = blockDim.x;
    uint8_t *dst = sm.at<uint8_t>(dst_off);
    const uint8_t *src = sm.at<uint8_t>(sm.src);
    int *winner = sm.at<int>(sm.off);
    const bool take_max = div_px < 0.0;  // ascending sweep: the largest source column writes last (:107)
    for (int c = tid; c < W; c += T_) winner[c] = take_max ? -1 : 0x7fffffff;
    __syncthreads();
    for (int col = tid; col < W; col += T_) {
        const double v = nds.get(col) * div_px + sep_px;
        if (!(v > -4.0e9 && v < 4.0e9)) continue;  // NaN / huge: int() gives INT64_MIN in the reference -> out of range
        const long long cd = (long long)col + (long long)v;  // int(): truncation toward zero
        if (cd >= 0 && cd < W) {
            if (take_max) atomicMax(&winner[(int)cd], col); else atomicMin(&winner[(int)cd], col);
        }
    }
    __syncthreads();
    // scattered (pre-fill) row -> dst for `none`, -> staging for the fills
    uint8_t *scat = (fill == DM_FILL_NONE) ? dst : sm.at<uint8_t>(sm.pm);
    for (int c = tid; c < W; c += T_) {
        const int wsrc = winner[c];
        const bool f = take_max ? (wsrc >= 0) : (wsrc != 0x7fffffff);
        uint8_t r = 0, g = 0, b = 0;
        if (f) { r = src[3 * wsrc]; g = src[3 * wsrc + 1]; b = src[3 * wsrc + 2]; }
        scat[3 * c] = r; scat[3 * c + 1] = g; scat[3 * c + 2] = b;
        winner[c] = f ? 1 : 0;  // from here on: the `filled` mask
    }
    __syncthreads();
    if (fill == DM_FILL_NONE) return;
    const int *filled = winner;
    if (fill == DM_FILL_NAIVE) {  // :142-157
        double adp = div_px < 0 ? -div_px : div_px;
        long long lim = (adp < 4.0e9) ? (long long)adp : 0;  // abs(int(div_px))
        for (int c = tid; c < W; c += T_) {
            int from = c;
            if (!filled[c]) {
                for (long long o = 1; o < lim + 2; ++o) {
                    const long long ro = c + o, lo = c - o;
                    if (ro < W && filled[ro]) { from = (int)ro; break; }
                    if (lo >= 0 && filled[lo]) { from = (int)lo; break; }
                    if (ro >= W && lo < 0) break;
                }
            }
            dst[3 * c] = scat[3 * from]; dst[3 * c + 1] = scat[3 * from + 1]; dst[3 * c + 2] = scat[3 * from + 2];
        }
        __syncthreads();
        return;
    }
    // naive_interpolating (:114-141) in closed form
    int *lastV = sm.at<int>(sm.cur), *nextV = sm.at<int>(sm.aux), *nextU = sm.at<int>(sm.off);  // nextU overwrites `filled` after it has been consumed
    for (int c = tid; c < W; c += T_) {
        const bool f = filled[c] != 0;
        const bool nonblack = ((int)scat[3 * c] + scat[3 * c + 1] + scat[3 * c + 2]) != 0;
        const bool V = f && nonblack;
        lastV[c] = V ? c : -1;
        nextV[c] = V ? c : W;
    }
    __syncthreads();
    for (int c = tid; c < W; c += T_) nextU[c] = filled[c] ? W : c;  // same thread reads and writes element c
    __syncthreads();
    block_scan_inclusive<int>(lastV, W, -1, OpMaxI(), false, sm.at<int>(sm.wtot_i));
    block_scan_inclusive<int>(nextV, W, W, OpMinI(), true, sm.at<int>(sm.wtot_i));
    block_scan_inclusive<int>(nextU, W, W, OpMinI(), true, sm.at<int>(sm.wtot_i));
    for (int p = tid; p < W; p += T_) {
        const int v = lastV[p];
        const int l = (v + 1 < W) ? nextU[v + 1] : W;
        uint8_t o0 = scat[3 * p], o1 = scat[3 * p + 1], o2 = scat[3 * p + 2];
        if (l <= p) {
            const int r = nextV[p];  // p itself is not V here
            int lb[3] = {0, 0, 0}, rb[3] = {0, 0, 0};
            if (l > 0) { lb[0] = scat[3 * (l - 1)]; lb[1] = scat[3 * (l - 1) + 1]; lb[2] = scat[3 * (l - 1) + 2]; }
            if (r < W) { rb[0] = scat[3 * r]; rb[1] = scat[3 * r + 1]; rb[2] = scat[3 * r + 2]; }
            if (lb[0] + lb[1] + lb[2] == 0) { lb[0] = rb[0]; lb[1] = rb[1]; lb[2] = rb[2]; }
            else if (rb[0] + rb[1] + rb[2] == 0) { rb[0] = lb[0]; rb[1] = lb[1]; rb[2] = lb[2]; }
            const double total_steps = (double)(1 + r - l);
            const double k = (double)(p - l + 1);
            o0 = (uint8_t)(lb[0] + f64_to_u8_wrap(((double)rb[0] - (double)lb[0]) / total_steps * k));
            o1 = (uint8_t)(lb[1] + f64_to_u8_wrap(((double)rb[1] - (double)lb[1]) / total_steps * k));
            o2 = (uint8_t)(lb[2] + f64_to_u8_wrap(((double)rb[2] - (double)lb[2]) / total_steps * k));
        }
        dst[3 * p] = o0; dst[3 * p + 1] = o1; dst[3 * p + 2] = o2;
    }
    __syncthreads();
}

template <bool POLY>
__global__ void __launch_bounds__(256, POLY ? 2 : 4) stereo_row_kernel(StereoArgs a, int pow_kind) {
    const int W = a.W, y = blockIdx.x, b = blockIdx.y;
    const int tid = threadIdx.x, T_ = blockDim.x;
    const bool poly = POLY;
    const int n = a.fill == DM_FILL_POLYLINES_SHARP ? 2 * W + 2 : W + 2;
    const bool u16 = a.depth_kind == DM_DEPTH_U16;

    RowSmem sm;
    uint32_t o = 0;
    auto carve = [&](size_t bytes) { const uint32_t p = o; o += (uint32_t)((bytes + 15) & ~(size_t)15); return p; };
    sm.wtot_d = carve(32 * sizeof(double));
    sm.wtot_i = carve(32 * sizeof(int));
    sm.ndp = carve(u16 ? sizeof(uint16_t) * W : sizeof(double) * W);   // u16 depth row, or the fp64 nd row
    sm.xs = carve(poly ? sizeof(double) * n : 16);
    sm.pm = carve(poly ? sizeof(double) * n : (size_t)3 * W);
    sm.off = carve(sizeof(int) * (W + 4));
    sm.cur = carve(a.fill == DM_FILL_NAIVE_INTERPOLATING ? sizeof(int) * (W + 3) : 16);
    sm.aux = carve(a.fill == DM_FILL_NAIVE_INTERPOLATING ? sizeof(int) * (W + 1) : 16);
    sm.order = carve(poly ? sizeof(uint16_t) * n : 16);
    sm.src = carve(poly ? (size_t)4 * W : (size_t)3 * W);
    sm.eye[0] = carve((size_t)3 * W);
    sm.eye[1] = carve((size_t)3 * W);
    // the naive family reads the row as bytes; polylines reads whole pixels (R | G << 8 | B << 16): the raw bytes land in the
    // left-eye staging row first and are packed from there
    uint8_t *s_src = sm.at<uint8_t>(poly ? sm.eye[0] : sm.src);
    uint32_t *s_px = sm.at<uint32_t>(sm.src);

    // ---- load the row: RGB bytes and nd ** exponent --------------------------------------------------------
    const uint8_t *src_g = a.rgb + ((int64_t)b * a.H + y) * (int64_t)W * 3;
    {
        const int nbytes = 3 * W;
        const int head = (int)((16 - ((uintptr_t)src_g & 15)) & 15);
        const int h = head < nbytes ? head : nbytes;
        for (int i = tid; i < h; i += T_) s_src[i] = __ldg(src_g + i);
        const int nvec = (nbytes - h) >> 4;
        for (int i = tid; i < nvec; i += T_) {
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(src_g + h) + i);
            uint8_t *d = s_src + h + i * 16;
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) { d[4 * k] = w[k] & 0xff; d[4 * k + 1] = (w[k] >> 8) & 0xff; d[4 * k + 2] = (w[k] >> 16) & 0xff; d[4 * k + 3] = w[k] >> 24; }
        }
        for (int i = h + nvec * 16 + tid; i < nbytes; i += T_) s_src[i] = __ldg(src_g + i);
    }
    if (POLY) {
        __syncthreads();
        for (int c = tid; c < W; c += T_) s_px[c] = (uint32_t)s_src[3 * c] | ((uint32_t)s_src[3 * c + 1] << 8) | ((uint32_t)s_src[3 * c + 2] << 16);
    }
    bool flat = false;
    NdSrc nds;
    nds.ndp = nullptr; nds.dep = nullptr; nds.mn = 0; nds.den = 1.0; nds.rden = 1.0; nds.expo = a.exponent; nds.pow_kind = pow_kind;
    if (u16) {
        const uint16_t *dep = (const uint16_t *)a.depth + ((int64_t)b * a.H + y) * (int64_t)W;
        const uint32_t mn = a.minmax[2 * b], mx = a.minmax[2 * b + 1];
        flat = (mx == mn);
        uint16_t *s_dep = sm.at<uint16_t>(sm.ndp);
        for (int c = tid; c < W; c += T_) s_dep[c] = __ldg(dep + c);
        nds.dep = s_dep; nds.mn = mn; nds.den = (double)(mx - mn); nds.rden = 1.0 / nds.den;   // :81 (d - min) / (max - min), float64 true-divide
    } else {
        const double *dep = (const double *)a.depth + ((int64_t)b * a.H + y) * (int64_t)W;
        double *s_ndp = sm.at<double>(sm.ndp);
        for (int c = tid; c < W; c += T_) s_ndp[c] = pow_ref(__ldg(dep + c), a.exponent, pow_kind);
        nds.ndp = s_ndp;
    }
    __syncthreads();

    // ---- eyes ---------------------------------------------------------------------------------------------------
    for (int e = 0; e < 2; ++e) {
        if (a.eye_mode[e] == DM_EYE_SKIP) continue;
        const uint32_t dst_off = e == 0 ? sm.eye[0] : sm.eye[1];
        uint8_t *dst = sm.at<uint8_t>(dst_off);
        if (a.eye_mode[e] == DM_EYE_IDENTITY) {
            if (POLY) { for (int i = tid; i < 3 * W; i += T_) dst[i] = (uint8_t)(s_px[i / 3] >> (8 * (i % 3))); }
            else { for (int i = tid; i < 3 * W; i += T_) dst[i] = s_src[i]; }
            __syncthreads();
        } else if (flat) {
            // max == min: nd is 0/0 = NaN everywhere.  Reference behaviour (pinned by the oracle): the naive family
            // scatters nothing (black row); polylines degenerates to the first pixel's colour across the row.
            for (int c = tid; c < W; c += T_)
                for (int k = 0; k < 3; ++k) dst[3 * c + k] = poly ? (uint8_t)(s_px[0] >> (8 * k)) : (uint8_t)0;
            __syncthreads();
        } else if (POLY) {
            if (a.fill == DM_FILL_POLYLINES_SHARP)
                polylines_eye<true>(sm, nds, W, a.div_px[e], a.sep_px[e], dst_off, (y == 0 && b == 0 && e == 0) ? a.dbg : nullptr);
            else
                polylines_eye<false>(sm, nds, W, a.div_px[e], a.sep_px[e], dst_off, (y == 0 && b == 0 && e == 0) ? a.dbg : nullptr);
        } else {
            naive_eye(sm, nds, W, a.div_px[e], a.sep_px[e], a.fill, dst_off);
        }
    }

    // ---- pack + store -------------------------------------------------------------------------------------------
    if (a.pack == DM_PACK_ANAGLYPH) {
        const uint8_t *er = sm.at<uint8_t>(a.red_eye ? sm.eye[1] : sm.eye[0]), *ec = sm.at<uint8_t>(a.red_eye ? sm.eye[0] : sm.eye[1]);
        uint8_t *comp = sm.at<uint8_t>(sm.src);      // the source row is dead by now
        __syncthreads();
        for (int c = tid; c < W; c += T_) { comp[3 * c] = er[3 * c]; comp[3 * c + 1] = ec[3 * c + 1]; comp[3 * c + 2] = ec[3 * c + 2]; }
        __syncthreads();
        store_row(a.out[0] + (int64_t)b * a.img_stride[0] + (int64_t)y * a.row_stride[0], comp, 3 * W);
    } else {
        for (int e = 0; e < 2; ++e) {
            if (a.eye_mode[e] == DM_EYE_SKIP || !a.out[e]) continue;
            store_row(a.out[e] + (int64_t)b * a.img_stride[e] + (int64_t)y * a.row_stride[e], sm.at<uint8_t>(e == 0 ? sm.eye[0] : sm.eye[1]), 3 * W);
        }
    }
}

__global__ void __launch_bounds__(256) minmax_u16_kernel(const uint16_t *__restrict__ depth, int64_t n, uint32_t *ws) {
    const int b = blockIdx.y;
    const uint16_t *p = depth + (int64_t)b * n;
    uint32_t lo = 0xffffffffu, hi = 0u;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    const bool vec = (n % 8 == 0) && (((uintptr_t)depth) % 16 == 0);
    if (vec) {
        const uint4 *p4 = reinterpret_cast<const uint4 *>(p);
        for (int64_t i = tid; i < n / 8; i += nthreads) {
            const uint4 v = __ldg(p4 + i);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t a0 = w[k] & 0xffffu, a1 = w[k] >> 16;
                lo = min(lo, min(a0, a1)); hi = max(hi, max(a0, a1));
            }
        }
    } else {
        for (int64_t i = tid; i < n; i += nthreads) { const uint32_t v = __ldg(p + i); lo = min(lo, v); hi = max(hi, v); }
    }
    lo = warp_min_u32(lo); hi = warp_max_u32(hi);
    __shared__ uint32_t slo[8], shi[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { slo[warp] = lo; shi[warp] = hi; }
    __syncthreads();
    if (warp == 0) {
        lo = lane < 8 ? slo[lane] : 0xffffffffu; hi = lane < 8 ? shi[lane] : 0u;
        lo = warp_min_u32(lo); hi = warp_max_u32(hi);
        if (lane == 0) { atomicMin(ws + 2 * b, lo); atomicMax(ws + 2 * b + 1, hi); }
    }
}

__global__ void minmax_u16_init_kernel(uint32_t *ws, int B) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) { ws[2 * i] = 0xffffffffu; ws[2 * i + 1] = 0u; }
}

static size_t stereo_smem_bytes(int W, int fill, int depth_kind) {
    const bool poly = fill == DM_FILL_POLYLINES_SOFT || fill == DM_FILL_POLYLINES_SHARP;
    const size_t n = fill == DM_FILL_POLYLINES_SHARP ? 2 * (size_t)W + 2 : (size_t)W + 2;
    auto r16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    const bool interp = fill == DM_FILL_NAIVE_INTERPOLATING;
    size_t s = r16(32 * 8) + r16(32 * 4) + r16((depth_kind == DM_DEPTH_U16 ? 2 : 8) * (size_t)W) + r16(poly ? 8 * n : 16) +
               r16(poly ? 8 * n : 3 * (size_t)W) + r16(4 * ((size_t)W + 4)) + r16(interp ? 4 * ((size_t)W + 3) : 16) +
               r16(interp ? 4 * ((size_t)W + 1) : 16) + r16(poly ? 2 * n : 16) + r16(poly ? 4 * (size_t)W : 3 * (size_t)W) + 2 * r16(3 * (size_t)W);
    return s;
}

}  // namespace dm

static double *g_stereo_dbg = nullptr;
// bring-up hook, not part of the C-ABI (hidden symbol): dumps the sorted vertex arrays of row 0 / image 0 / first warped eye
extern "C" void dm_stereo_set_debug_buffer(double *dev_buf) { g_stereo_dbg = dev_buf; }

extern "C" __attribute__((visibility("default"))) size_t dm_stereo_workspace_bytes(int B, int H, int W) {
    (void)H; (void)W;
    return dm::align_up((size_t)(B > 0 ? B : 1) * 2 * sizeof(uint32_t), 256);
}

extern "C" __attribute__((visibility("default"))) int dm_stereo(const uint8_t *rgb, const void *depth, int B, int H, int W, const dm_stereo_params *p,
                         uint8_t *out0, uint8_t *out1, void *workspace, size_t workspace_bytes, void *stream_) {
    using namespace dm;
    if (!rgb || !depth || !p || B <= 0 || H <= 0 || W <= 0) { set_error("dm_stereo: bad arguments"); return DM_E_INVALID; }
    if (p->fill < DM_FILL_NONE || p->fill > DM_FILL_POLYLINES_SHARP) { set_error("dm_stereo: unknown fill %d", p->fill); return DM_E_INVALID; }
    if (p->pack != DM_PACK_STRIDED && p->pack != DM_PACK_ANAGLYPH) { set_error("dm_stereo: unknown pack %d", p->pack); return DM_E_INVALID; }
    if (p->depth_kind != DM_DEPTH_U16 && p->depth_kind != DM_DEPTH_ND64) { set_error("dm_stereo: unknown depth_kind"); return DM_E_INVALID; }
    if (!out0 && (p->pack == DM_PACK_ANAGLYPH || p->eye_mode[0] != DM_EYE_SKIP)) { set_error("dm_stereo: out0 is NULL"); return DM_E_INVALID; }
    if (p->pack == DM_PACK_STRIDED && !out1 && p->eye_mode[1] != DM_EYE_SKIP) { set_error("dm_stereo: out1 is NULL"); return DM_E_INVALID; }
    if (p->pack == DM_PACK_ANAGLYPH && (p->eye_mode[0] == DM_EYE_SKIP || p->eye_mode[1] == DM_EYE_SKIP)) { set_error("dm_stereo: anaglyph needs both eyes"); return DM_E_INVALID; }
    if (H > 2147483647 / 1 || B > 65535) { set_error("dm_stereo: batch too large"); return DM_E_UNSUPPORTED; }
    if (W > 32000) { set_error("dm_stereo: rows wider than 32000 px are not supported"); return DM_E_UNSUPPORTED; }
    if (!workspace || workspace_bytes < dm_stereo_workspace_bytes(B, H, W)) { set_error("dm_stereo: workspace too small"); return DM_E_WORKSPACE; }
    cudaStream_t stream = (cudaStream_t)stream_;
    uint32_t *ws = (uint32_t *)workspace;

    const size_t smem = stereo_smem_bytes(W, p->fill, p->depth_kind);
    const bool poly = p->fill == DM_FILL_POLYLINES_SOFT || p->fill == DM_FILL_POLYLINES_SHARP;
    if (smem > 227 * 1024) {
        set_error("dm_stereo: a %d px row needs %zu B of shared memory (> 227 KB); image too wide for this fill mode", W, smem);
        return DM_E_UNSUPPORTED;
    }
    if (smem > 48 * 1024) {
        static PerDeviceFlag configured;
        if (!configured.test_and_set()) {
            DM_CUDA_CHECK(cudaFuncSetAttribute(stereo_row_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024)));
            DM_CUDA_CHECK(cudaFuncSetAttribute(stereo_row_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024)));
        }
    }
    if (p->depth_kind == DM_DEPTH_U16) {
        const int64_t n = (int64_t)H * W;
        minmax_u16_init_kernel<<<(B + 255) / 256, 256, 0, stream>>>(ws, B);
        DM_LAUNCH_CHECK("minmax_u16_init_kernel");
        int bx = (int)((n / 8 + 255) / 256);
        bx = bx < 1 ? 1 : (bx > 132 * 4 ? 132 * 4 : bx);
        minmax_u16_kernel<<<dim3(bx, B), 256, 0, stream>>>((const uint16_t *)depth, n, ws);
        DM_LAUNCH_CHECK("minmax_u16_kernel");
    }
    StereoArgs a;
    memset(&a, 0, sizeof(a));
    a.rgb = rgb; a.depth = depth; a.minmax = ws; a.H = H; a.W = W; a.exponent = p->exponent;
    for (int e = 0; e < 2; ++e) {
        a.div_px[e] = p->div_px[e]; a.sep_px[e] = p->sep_px[e]; a.eye_mode[e] = p->eye_mode[e];
        a.row_stride[e] = p->dst_row_stride[e]; a.img_stride[e] = p->dst_img_stride[e];
    }
    a.fill = p->fill; a.pack = p->pack; a.red_eye = p->anaglyph_red_eye ? 1 : 0; a.depth_kind = p->depth_kind;
    a.out[0] = out0; a.out[1] = out1;
    a.dbg = g_stereo_dbg;
    const int pow_kind = p->exponent == 1.0 ? 0 : (p->exponent == 2.0 ? 1 : 2);
    const int threads = W <= 256 ? 128 : 256;
    if (poly) stereo_row_kernel<true><<<dim3(H, B), threads, smem, stream>>>(a, pow_kind);
    else stereo_row_kernel<false><<<dim3(H, B), threads, smem, stream>>>(a, pow_kind);
    DM_LAUNCH_CHECK("stereo_row_kernel");
    return DM_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// dm_stereo_pack — the packings of create_stereoimages (src/stereoimage_generation.py:56-73) from a side-by-side pair, for
// requests with several modes: the eyes are computed once (left | right), every further mode is one byte-shuffling pass.
// dm_depth_to_nd64 — apply_stereo_divergence's normalisation (:79-81) for depth maps that are not uint16: numpy evaluates
// (d - min) / (max - min) in the array's own dtype (float32 stays float32, integers true-divide to float64); the result is
// widened to the float64 the row kernels read.
// ---------------------------------------------------------------------------------------------------------------------
namespace dm {

__global__ void __launch_bounds__(256) stereo_pack_kernel(const uint8_t *__restrict__ sbs, int H, int W, int mode, uint8_t *__restrict__ out) {
    // one thread per output pixel; blockIdx.y = output row, blockIdx.z = image
    const int b = blockIdx.z;
    const uint8_t *L = sbs + (size_t)b * H * 2 * W * 3;      // row y: [left eye W px | right eye W px]
    int oh = H, ow = W;
    if (mode == 0 || mode == 1) ow = 2 * W;
    if (mode == 2 || mode == 3) oh = 2 * H;
    const int y = blockIdx.y, x = blockIdx.x * 256 + threadIdx.x;
    if (x >= ow || y >= oh) return;
    int sy = y, sxr = x, sxg = x;     // source column (in the 2W-wide pair) of the red and of the green / blue channel
    switch (mode) {
        case 0: break;                                                        // left-right
        case 1: sxr = sxg = x < W ? x + W : x - W; break;                       // right-left
        case 2: sy = y < H ? y : y - H; sxr = sxg = y < H ? x : x + W; break;   // top-bottom: left eye on top
        case 3: sy = y < H ? y : y - H; sxr = sxg = y < H ? x + W : x; break;   // bottom-top
        case 4: sxr = x; sxg = x + W; break;                                    // red-cyan anaglyph: R from the left eye, G B from the right
        case 5: break;                                                        // left-only
        case 6: sxr = sxg = x + W; break;                                       // only-right
        default: sxr = x + W; sxg = x; break;                                   // cyan-red reverse anaglyph
    }
    const uint8_t *pr = L + ((size_t)sy * 2 * W + sxr) * 3, *pg = L + ((size_t)sy * 2 * W + sxg) * 3;
    uint8_t *o = out + (((size_t)b * oh + y) * ow + x) * 3;
    o[0] = pr[0]; o[1] = pg[1]; o[2] = pg[2];
}

template <typename T> struct NdTraits;
template <> struct NdTraits<float> {
    __device__ static bool less(float a, float b) { return a < b; }
    __device__ static double norm(float x, float mn, float mx) { return (double)__fdiv_rn(__fsub_rn(x, mn), __fsub_rn(mx, mn)); }
};
template <> struct NdTraits<double> {
    __device__ static bool less(double a, double b) { return a < b; }
    __device__ static double norm(double x, double mn, double mx) { return __ddiv_rn(__dsub_rn(x, mn), __dsub_rn(mx, mn)); }
};
template <> struct NdTraits<long long> {
    __device__ static bool less(long long a, long long b) { return a < b; }
    __device__ static double norm(long long x, long long mn, long long mx) { return __ddiv_rn((double)(x - mn), (double)(mx - mn)); }
};

// one CTA per image (these maps are small next to the network; the uint16 fast path does not come here)
template <typename T>
__global__ void __launch_bounds__(1024) depth_to_nd64_kernel(const T *__restrict__ depth, long long n, double *__restrict__ nd, int32_t *flat) {
    __shared__ T s_lo[32], s_hi[32];
    const int b = blockIdx.x;
    const T *p = depth + (size_t)b * n;
    T lo = p[0], hi = p[0];
    for (long long i = threadIdx.x; i < n; i += blockDim.x) { const T v = p[i]; if (NdTraits<T>::less(v, lo)) lo = v; if (NdTraits<T>::less(hi, v)) hi = v; }
    // NaNs: numpy's min / max propagate NaN; a NaN depth map is outside what the reference can render either — not reproduced
    for (int o = 16; o > 0; o >>= 1) {
        const T a = __shfl_xor_sync(0xffffffffu, lo, o), c = __shfl_xor_sync(0xffffffffu, hi, o);
        if (NdTraits<T>::less(a, lo)) lo = a;
        if (NdTraits<T>::less(hi, c)) hi = c;
    }
    if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    lo = s_lo[0]; hi = s_hi[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { if (NdTraits<T>::less(s_lo[w], lo)) lo = s_lo[w]; if (NdTraits<T>::less(hi, s_hi[w])) hi = s_hi[w]; }
    if (threadIdx.x == 0 && flat) flat[b] = (lo == hi) ? 1 : 0;
    double *o = nd + (size_t)b * n;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) o[i] = NdTraits<T>::norm(p[i], lo, hi);
}

}  // namespace dm

extern "C" __attribute__((visibility("default"))) int dm_stereo_pack(const uint8_t *sbs, int B, int H, int W, int mode, uint8_t *out, void *stream_) {
    using namespace dm;
    if (!sbs || !out || B <= 0 || H <= 0 || W <= 0 || mode < 0 || mode > 7) { set_error("dm_stereo_pack: bad arguments"); return DM_E_INVALID; }
    const int oh = (mode == 2 || mode == 3) ? 2 * H : H, ow = (mode == 0 || mode == 1) ? 2 * W : W;
    if (oh > 65535 || B > 65535) { set_error("dm_stereo_pack: shape too large"); return DM_E_UNSUPPORTED; }
    stereo_pack_kernel<<<dim3((unsigned)((ow + 255) / 256), (unsigned)oh, (unsigned)B), 256, 0, (cudaStream_t)stream_>>>(sbs, H, W, mode, out);
    DM_LAUNCH_CHECK("stereo_pack_kernel");
    return DM_OK;
}

/* dtype: 0 float32, 1 float64, 2 int64.  nd_out float64 [B, n]; flat_out (optional) int32[B]: 1 where max == min */
extern "C" __attribute__((visibility("default"))) int dm_depth_to_nd64(const void *depth, int dtype, int B, long long n, double *nd_out, int32_t *flat_out,
                                                                    void *stream_) {
    using namespace dm;
    if (!depth || !nd_out || B <= 0 || n <= 0) { set_error("dm_depth_to_nd64: bad arguments"); return DM_E_INVALID; }
    cudaStream_t st = (cudaStream_t)stream_;
    if (dtype == 0) depth_to_nd64_kernel<float><<<B, 1024, 0, st>>>((const float *)depth, n, nd_out, flat_out);
    else if (dtype == 1) depth_to_nd64_kernel<double><<<B, 1024, 0, st>>>((const double *)depth, n, nd_out, flat_out);
    else if (dtype == 2) depth_to_nd64_kernel<long long><<<B, 1024, 0, st>>>((const long long *)depth, n, nd_out, flat_out);
    else { set_error("dm_depth_to_nd64: dtype %d unsupported", dtype); return DM_E_UNSUPPORTED; }
    DM_LAUNCH_CHECK("depth_to_nd64_kernel");
    return DM_OK;
}
