// N1 — prediction -> 16-bit depth.  Replaces src/core.py:189-211 (model branch) + convert_to_i16 (src/core.py:44-50).
//
// Two launches per batch, both HBM-bound:
//   minmax_f32_kernel : exact per-image min / max (order-preserving integer atomics), 4 B/px read
//   quantize_kernel   : invert, normalise, optional "Range" clip, *65536 + 1e-4, clip, truncate; 4 B/px read, 2 B/px write
// float32 arithmetic with explicit round-to-nearest intrinsics (no FMA contraction), mirroring numpy's float32 ops.
// "Range" clip needs no second reduction: t(x) = (x-lo)/(hi-lo) is monotone non-decreasing in floating point, so the
// min / max of clip(t, far, near) are clip(t(lo)) = clip(0) and clip(t(hi)) = clip(1).
#include "common.cuh"

namespace dm {

__global__ void minmax_init_kernel(uint32_t *ws, int B) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) { ws[2 * i] = 0xffffffffu; ws[2 * i + 1] = 0u; }
}

__global__ void __launch_bounds__(256) minmax_f32_kernel(const float *__restrict__ pred, int64_t n, uint32_t *ws, int vec_ok) {
    const int b = blockIdx.y;
    const float *p = pred + (int64_t)b * n;
    uint32_t lo = 0xffffffffu, hi = 0u;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (vec_ok) {
        const float4 *p4 = reinterpret_cast<const float4 *>(p);
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += nthreads) {
            float4 v = __ldg(p4 + i);
            uint32_t a = f32_to_ordered(v.x), c = f32_to_ordered(v.y), d = f32_to_ordered(v.z), e = f32_to_ordered(v.w);
            lo = min(lo, min(min(a, c), min(d, e)));
            hi = max(hi, max(max(a, c), max(d, e)));
        }
    } else {
        for (int64_t i = tid; i < n; i += nthreads) {
            uint32_t a = f32_to_ordered(__ldg(p + i));
            lo = min(lo, a);
            hi = max(hi, a);
        }
    }
    lo = warp_min_u32(lo);
    hi = warp_max_u32(hi);
    __shared__ uint32_t slo[8], shi[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { slo[warp] = lo; shi[warp] = hi; }
    __syncthreads();
    if (warp == 0) {
        lo = lane < (blockDim.x >> 5) ? slo[lane] : 0xffffffffu;
        hi = lane < (blockDim.x >> 5) ? shi[lane] : 0u;
        lo = warp_min_u32(lo);
        hi = warp_max_u32(hi);
        if (lane == 0) { atomicMin(ws + 2 * b, lo); atomicMax(ws + 2 * b + 1, hi); }
    }
}

struct QuantParams {
    int invert, clip_mode;
    float clip_far, clip_near;
};

__device__ __forceinline__ uint16_t quantize_one(float x, float lo, float den, int invert, int clip_mode, float cf,
                                                 float cn, float lo2, float den2) {
    float xp = invert ? __fmul_rn(x, -1.0f) : x;
    float t = __fdiv_rn(__fsub_rn(xp, lo), den);
    if (clip_mode == 1) {
        t = fminf(fmaxf(t, cf), cn);
        t = __fdiv_rn(__fsub_rn(t, lo2), den2);
    }
    float q = __fadd_rn(__fmul_rn(t, 65536.0f), 0.0001f);
    q = fminf(fmaxf(q, 0.0f), 65535.8984375f);  // float32(65536 - 0.1)
    if (!(q == q)) q = 0.0f;
    return (uint16_t)(int)q;
}

__global__ void __launch_bounds__(256) quantize_kernel(const float *__restrict__ pred, int64_t n, const uint32_t *__restrict__ ws,
                                                       QuantParams qp, uint16_t *__restrict__ out, int32_t *degenerate, int vec_ok) {
    const int b = blockIdx.y;
    const float *p = pred + (int64_t)b * n;
    uint16_t *o = out + (int64_t)b * n;
    const float mn = ordered_to_f32(ws[2 * b]), mx = ordered_to_f32(ws[2 * b + 1]);
    // src/core.py:189  abs(max - min) > np.finfo("float").eps   (float32 difference vs float64 epsilon)
    const bool ok = fabs((double)__fsub_rn(mx, mn)) > 2.220446049250313e-16;
    if (degenerate && blockIdx.x == 0 && threadIdx.x == 0) degenerate[b] = ok ? 0 : 1;
    const float lo = qp.invert ? __fmul_rn(mx, -1.0f) : mn;
    const float hi = qp.invert ? __fmul_rn(mn, -1.0f) : mx;
    const float den = __fsub_rn(hi, lo);
    float lo2 = 0.f, den2 = 1.f;
    if (qp.clip_mode == 1) {
        float t_lo = __fdiv_rn(__fsub_rn(lo, lo), den), t_hi = __fdiv_rn(__fsub_rn(hi, lo), den);
        lo2 = fminf(fmaxf(t_lo, qp.clip_far), qp.clip_near);
        float hi2 = fminf(fmaxf(t_hi, qp.clip_far), qp.clip_near);
        den2 = __fsub_rn(hi2, lo2);
    }
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (vec_ok) {
        const float4 *p4 = reinterpret_cast<const float4 *>(p);
        ushort4 *o4 = reinterpret_cast<ushort4 *>(o);
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += nthreads) {
            ushort4 r = make_ushort4(0, 0, 0, 0);
            if (ok) {
                float4 v = __ldg(p4 + i);
                r.x = quantize_one(v.x, lo, den, qp.invert, qp.clip_mode, qp.clip_far, qp.clip_near, lo2, den2);
                r.y = quantize_one(v.y, lo, den, qp.invert, qp.clip_mode, qp.clip_far, qp.clip_near, lo2, den2);
                r.z = quantize_one(v.z, lo, den, qp.invert, qp.clip_mode, qp.clip_far, qp.clip_near, lo2, den2);
                r.w = quantize_one(v.w, lo, den, qp.invert, qp.clip_mode, qp.clip_far, qp.clip_near, lo2, den2);
            }
            o4[i] = r;
        }
    } else {
        for (int64_t i = tid; i < n; i += nthreads)
            o[i] = ok ? quantize_one(__ldg(p + i), lo, den, qp.invert, qp.clip_mode, qp.clip_far, qp.clip_near, lo2, den2) : (uint16_t)0;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// "Outliers" clip (src/core.py:200-202): fb, nb = np.percentile(out, [far*100, near*100]); out = np.clip(out, fb, nb).
// np.percentile (method "linear") needs, per percentile, the two order statistics around the virtual index and a float64
// interpolation weight; from there on numpy works in FLOAT64 (percentile returns float64 scalars, so np.clip promotes the
// float32 image).  The order statistics are found exactly by a 4-pass, 8-bit radix select on the order-preserving integer
// image of the (sign-applied) values: each pass histograms the digit of the elements that still match each target's
// prefix, a 4-warp kernel picks the digit that contains the wanted rank.  Ranks and weights are computed by the host
// face with numpy's own expression (they depend only on H*W and the two fractions).
// ---------------------------------------------------------------------------------------------------------------------
struct SelectState {          // per image
    uint32_t prefix[4];       // key bits decided so far, per target
    uint32_t rank[4];         // rank still to be found inside the matching subset
    uint32_t hist[4][256];
};

__global__ void select_init_kernel(SelectState *st, int B, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    const int b = blockIdx.x;
    if (b >= B) return;
    SelectState &s = st[b];
    if (threadIdx.x < 4) {
        s.prefix[threadIdx.x] = 0u;
        s.rank[threadIdx.x] = threadIdx.x == 0 ? r0 : (threadIdx.x == 1 ? r1 : (threadIdx.x == 2 ? r2 : r3));
    }
    for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&s.hist[0][0])[i] = 0u;
}

__global__ void __launch_bounds__(256) select_hist_kernel(const float *__restrict__ pred, int64_t n, int invert, int pass, SelectState *st) {
    __shared__ uint32_t h[4][256];
    const int b = blockIdx.y;
    const float *p = pred + (int64_t)b * n;
    for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&h[0][0])[i] = 0u;
    const int shift = 24 - 8 * pass;
    const uint32_t mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    uint32_t pre[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) pre[t] = st[b].prefix[t];
    __syncthreads();
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = tid; i < n; i += nthreads) {
        const float x = __ldg(p + i);
        const uint32_t key = f32_to_ordered(invert ? __fmul_rn(x, -1.0f) : x);
        const uint32_t digit = (key >> shift) & 255u;
        const uint32_t hi = key & mask;
        // the two ranks of one percentile (and often all four) share their prefix: count once, add to each matching target
        if (hi == pre[0]) atomicAdd(&h[0][digit], 1u);
        if (hi == pre[1]) atomicAdd(&h[1][digit], 1u);
        if (hi == pre[2]) atomicAdd(&h[2][digit], 1u);
        if (hi == pre[3]) atomicAdd(&h[3][digit], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
        const uint32_t v = (&h[0][0])[i];
        if (v) atomicAdd(&st[b].hist[0][0] + i, v);
    }
}

// one warp per target: find the digit whose cumulative count crosses the wanted rank, descend into it
__global__ void __launch_bounds__(128) select_pick_kernel(SelectState *st, int pass) {
    const int b = blockIdx.x, t = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SelectState &s = st[b];
    const int shift = 24 - 8 * pass;
    uint32_t c[8], sum = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i] = s.hist[t][lane * 8 + i]; sum += c[i]; }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    const uint32_t excl = incl - sum;
    const uint32_t want = s.rank[t];
    const bool mine = want >= excl && want < incl;      // exactly one lane (the counts add up to the subset size > want)
    __syncwarp();
    if (mine) {
        uint32_t run = excl;
        int digit = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (want >= run && want < run + c[i]) { digit = lane * 8 + i; break; }
            run += c[i];
        }
        s.prefix[t] |= (uint32_t)digit << shift;
        s.rank[t] = want - run;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s.hist[t][lane * 8 + i] = 0u;
}

struct OutlierParams {
    int invert;
    double gamma_far, gamma_near;     // np.percentile interpolation weights
};

__global__ void __launch_bounds__(256) quantize_outliers_kernel(const float *__restrict__ pred, int64_t n, const uint32_t *__restrict__ ws,
                                                                const SelectState *__restrict__ st, OutlierParams op,
                                                                uint16_t *__restrict__ out, int32_t *degenerate) {
    const int b = blockIdx.y;
    const float *p = pred + (int64_t)b * n;
    uint16_t *o = out + (int64_t)b * n;
    const float mn = ordered_to_f32(ws[2 * b]), mx = ordered_to_f32(ws[2 * b + 1]);
    const bool ok = fabs((double)__fsub_rn(mx, mn)) > 2.220446049250313e-16;      // src/core.py:189
    if (degenerate && blockIdx.x == 0 && threadIdx.x == 0) degenerate[b] = ok ? 0 : 1;
    // numpy _lerp(a, b, t): diff = b - a in float32; t < 0.5: a + diff * t, else b - diff * (1 - t), in float64
    auto lerp = [](float a, float bb, double t) {
        const double diff = (double)__fsub_rn(bb, a);
        return t >= 0.5 ? __dsub_rn((double)bb, __dmul_rn(diff, __dsub_rn(1.0, t))) : __dadd_rn((double)a, __dmul_rn(diff, t));
    };
    const double fb = lerp(ordered_to_f32(st[b].prefix[0]), ordered_to_f32(st[b].prefix[1]), op.gamma_far);
    const double nb = lerp(ordered_to_f32(st[b].prefix[2]), ordered_to_f32(st[b].prefix[3]), op.gamma_near);
    const float lo_f = op.invert ? __fmul_rn(mx, -1.0f) : mn, hi_f = op.invert ? __fmul_rn(mn, -1.0f) : mx;
    // np.clip = minimum(maximum(x, fb), nb); it is monotone, so the extremes of the clipped image are the clipped extremes
    const double lo = fmin(fmax((double)lo_f, fb), nb), hi = fmin(fmax((double)hi_f, fb), nb);
    const double den = __dsub_rn(hi, lo);
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = tid; i < n; i += nthreads) {
        uint16_t r = 0;
        if (ok) {
            const float x = __ldg(p + i);
            const double v = fmin(fmax((double)(op.invert ? __fmul_rn(x, -1.0f) : x), fb), nb);
            double q = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(v, lo), den), 65536.0), 0.0001);
            q = fmin(fmax(q, 0.0), 65535.9);
            r = (q == q) ? (uint16_t)(int)q : (uint16_t)0;        // 0/0 when the clip collapses the range: numpy's NaN -> 0
        }
        o[i] = r;
    }
}

}  // namespace dm

extern "C" __attribute__((visibility("default"))) size_t dm_normalize_u16_workspace_bytes(int B) { return dm::align_up((size_t)(B > 0 ? B : 1) * 2 * sizeof(uint32_t), 256); }

extern "C" __attribute__((visibility("default"))) int dm_normalize_u16(const float *pred, int B, int H, int W, int invert, int clip_mode, float clip_far,
                                float clip_near, uint16_t *depth_out, int32_t *degenerate_flags, void *workspace,
                                size_t workspace_bytes, void *stream_) {
    using namespace dm;
    if (!pred || !depth_out || B <= 0 || H <= 0 || W <= 0) { set_error("dm_normalize_u16: bad arguments"); return DM_E_INVALID; }
    if (clip_mode != 0 && clip_mode != 1) { set_error("dm_normalize_u16: clip_mode %d unsupported", clip_mode); return DM_E_UNSUPPORTED; }
    if (!workspace || workspace_bytes < dm_normalize_u16_workspace_bytes(B)) { set_error("dm_normalize_u16: workspace too small"); return DM_E_WORKSPACE; }
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t n = (int64_t)H * W;
    uint32_t *ws = (uint32_t *)workspace;
    const int vec_ok = (n % 4 == 0) && (((uintptr_t)pred) % 16 == 0) && (((uintptr_t)depth_out) % 8 == 0);
    minmax_init_kernel<<<(B + 255) / 256, 256, 0, stream>>>(ws, B);
    DM_LAUNCH_CHECK("minmax_init_kernel");
    int64_t work = vec_ok ? n / 4 : n;
    int bx = (int)((work + 256 * 4 - 1) / (256 * 4));
    if (bx < 1) bx = 1;
    if (bx > 132 * 8) bx = 132 * 8;
    dim3 grid(bx, B);
    minmax_f32_kernel<<<grid, 256, 0, stream>>>(pred, n, ws, vec_ok);
    DM_LAUNCH_CHECK("minmax_f32_kernel");
    QuantParams qp{invert ? 1 : 0, clip_mode, clip_far, clip_near};
    quantize_kernel<<<grid, 256, 0, stream>>>(pred, n, ws, qp, depth_out, degenerate_flags, vec_ok);
    DM_LAUNCH_CHECK("quantize_kernel");
    return DM_OK;
}

extern "C" __attribute__((visibility("default"))) size_t dm_normalize_u16_outliers_workspace_bytes(int B) {
    const size_t b = (size_t)(B > 0 ? B : 1);
    return dm::align_up(b * 2 * sizeof(uint32_t), 256) + dm::align_up(b * sizeof(dm::SelectState), 256);
}

extern "C" __attribute__((visibility("default"))) int dm_normalize_u16_outliers(const float *pred, int B, int H, int W, int invert, const int64_t ranks[4],
                                         double gamma_far, double gamma_near, uint16_t *depth_out, int32_t *degenerate_flags,
                                         void *workspace, size_t workspace_bytes, void *stream_) {
    using namespace dm;
    if (!pred || !depth_out || !ranks || B <= 0 || H <= 0 || W <= 0) { set_error("dm_normalize_u16_outliers: bad arguments"); return DM_E_INVALID; }
    const int64_t n = (int64_t)H * W;
    for (int i = 0; i < 4; ++i)
        if (ranks[i] < 0 || ranks[i] >= n || n >= (1ll << 32)) { set_error("dm_normalize_u16_outliers: rank %d out of range", i); return DM_E_INVALID; }
    if (!workspace || workspace_bytes < dm_normalize_u16_outliers_workspace_bytes(B)) { set_error("dm_normalize_u16_outliers: workspace too small"); return DM_E_WORKSPACE; }
    cudaStream_t stream = (cudaStream_t)stream_;
    uint32_t *ws = (uint32_t *)workspace;
    SelectState *st = (SelectState *)((uint8_t *)workspace + align_up((size_t)B * 2 * sizeof(uint32_t), 256));
    const int vec_ok = (n % 4 == 0) && (((uintptr_t)pred) % 16 == 0);
    minmax_init_kernel<<<(B + 255) / 256, 256, 0, stream>>>(ws, B);
    DM_LAUNCH_CHECK("minmax_init_kernel");
    int64_t work = vec_ok ? n / 4 : n;
    int bx = (int)((work + 256 * 4 - 1) / (256 * 4));
    if (bx < 1) bx = 1;
    if (bx > 132 * 8) bx = 132 * 8;
    dim3 grid(bx, B);
    minmax_f32_kernel<<<grid, 256, 0, stream>>>(pred, n, ws, vec_ok);
    DM_LAUNCH_CHECK("minmax_f32_kernel");
    select_init_kernel<<<B, 256, 0, stream>>>(st, B, (uint32_t)ranks[0], (uint32_t)ranks[1], (uint32_t)ranks[2], (uint32_t)ranks[3]);
    DM_LAUNCH_CHECK("select_init_kernel");
    int sx = (int)((n + 256 * 16 - 1) / (256 * 16));
    if (sx < 1) sx = 1;
    if (sx > 132 * 4) sx = 132 * 4;
    for (int pass = 0; pass < 4; ++pass) {
        select_hist_kernel<<<dim3(sx, B), 256, 0, stream>>>(pred, n, invert ? 1 : 0, pass, st);
        DM_LAUNCH_CHECK("select_hist_kernel");
        select_pick_kernel<<<B, 128, 0, stream>>>(st, pass);
        DM_LAUNCH_CHECK("select_pick_kernel");
    }
    OutlierParams op{invert ? 1 : 0, gamma_far, gamma_near};
    quantize_outliers_kernel<<<grid, 256, 0, stream>>>(pred, n, ws, st, op, depth_out, degenerate_flags);
    DM_LAUNCH_CHECK("quantize_outliers_kernel");
    return DM_OK;
}

// =====================================================================================================================
// §8(f) rank 1 — video mode's cross-frame normalisation.  Replaces src/video_mode.py:103-128 (process_predicitons).
//   'none'          every frame scaled with the GLOBAL float32 min / max over all frames: one min/max reduction (an
//                   all-reduce(MIN/MAX) of two floats when the frames are sharded over GPUs) + one scaling pass;
//   'experimental'  the 0.5 / 99.5 percentiles of a 5-tap temporal blend (0.1 0.2 0.4 0.2 0.1, frame indices clamped) give
//                   the bounds; the ORIGINAL frames are scaled in float64, unclipped.  The percentiles are found with the
//                   exact radix select above run over the whole blended stack; when frames are sharded, the four
//                   256-bin histograms of a pass are summed across ranks (an all-reduce of 4 KB) before the digit pick.
// Every step is its own entry point so the host can put the collective between them; nothing synchronises with the host.
// =====================================================================================================================
namespace dm {

__global__ void __launch_bounds__(256) video_blend_kernel(const float *__restrict__ frames, int64_t hw, int base_global, int n_total,
                                                          int out_first, int out_count, float *__restrict__ out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)out_count * hw) return;
    const int i = (int)(idx / hw);
    const int64_t px = idx - (int64_t)i * hw;
    const int g = out_first + i;
    const float taps[5] = {0.10f, 0.20f, 0.40f, 0.20f, 0.10f};       // float32(mul) * float32 frame, accumulated in float32
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 5; ++u) {
        int k = g + u - 2;
        k = k < 0 ? 0 : (k > n_total - 1 ? n_total - 1 : k);
        acc = __fadd_rn(acc, __fmul_rn(taps[u], __ldg(frames + (int64_t)(k - base_global) * hw + px)));
    }
    out[idx] = acc;
}

__global__ void video_minmax_export_kernel(const uint32_t *ws, float *out2) {
    if (threadIdx.x == 0) { out2[0] = ordered_to_f32(ws[0]); out2[1] = ordered_to_f32(ws[1]); }
}

__global__ void __launch_bounds__(256) video_scale_f32_kernel(const float *__restrict__ x, int64_t n, const float *__restrict__ lohi, float *__restrict__ out) {
    const float lo = lohi[0], den = __fsub_rn(lohi[1], lohi[0]);
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += nthreads) out[i] = __fdiv_rn(__fsub_rn(__ldg(x + i), lo), den);
}

__global__ void video_bounds_kernel(const SelectState *st, double gamma_lo, double gamma_hi, double *ab) {
    if (threadIdx.x != 0) return;
    auto lerp = [](float a, float bb, double t) {     // numpy _lerp, as in quantize_outliers_kernel
        const double diff = (double)__fsub_rn(bb, a);
        return t >= 0.5 ? __dsub_rn((double)bb, __dmul_rn(diff, __dsub_rn(1.0, t))) : __dadd_rn((double)a, __dmul_rn(diff, t));
    };
    ab[0] = lerp(ordered_to_f32(st->prefix[0]), ordered_to_f32(st->prefix[1]), gamma_lo);
    ab[1] = lerp(ordered_to_f32(st->prefix[2]), ordered_to_f32(st->prefix[3]), gamma_hi);
}

__global__ void __launch_bounds__(256) video_scale_f64_kernel(const float *__restrict__ x, int64_t n, const double *__restrict__ ab, double *__restrict__ out) {
    const double a = ab[0], den = __dsub_rn(ab[1], ab[0]);
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += nthreads) out[i] = __ddiv_rn(__dsub_rn((double)__ldg(x + i), a), den);
}

static int video_grid(int64_t n) {
    int64_t b = (n + 256 * 8 - 1) / (256 * 8);
    return (int)(b < 1 ? 1 : (b > 132 * 8 ? 132 * 8 : b));
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

DM_EXPORT size_t dm_video_workspace_bytes(void) { return dm::align_up(sizeof(dm::SelectState), 256) + 256; }

/* frames: fp32 [count, hw] = global frames [base_global, base_global + count); out: blended global frames [out_first, out_first + out_count) */
DM_EXPORT int dm_video_blend(const float *frames, long long hw, int base_global, int count, int n_total, int out_first, int out_count, float *out, void *stream_) {
    using namespace dm;
    if (!frames || !out || hw <= 0 || count <= 0 || n_total <= 0 || out_count <= 0) { set_error("dm_video_blend: bad arguments"); return DM_E_INVALID; }
    const int lo = out_first - 2 < 0 ? 0 : out_first - 2, hi = out_first + out_count + 1 > n_total - 1 ? n_total - 1 : out_first + out_count + 1;
    if (lo < base_global || hi > base_global + count - 1) { set_error("dm_video_blend: the local frames do not cover the two-frame halo"); return DM_E_INVALID; }
    const int64_t total = (int64_t)out_count * hw;
    video_blend_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(frames, hw, base_global, n_total, out_first, out_count, out);
    DM_LAUNCH_CHECK("video_blend_kernel");
    return DM_OK;
}

/* exact float32 min / max of x[0..n) -> lohi_out[2] (device) */
DM_EXPORT int dm_video_minmax(const float *x, long long n, float *lohi_out, void *workspace, size_t workspace_bytes, void *stream_) {
    using namespace dm;
    if (!x || !lohi_out || n <= 0 || !workspace || workspace_bytes < dm_video_workspace_bytes()) { set_error("dm_video_minmax: bad arguments"); return DM_E_INVALID; }
    cudaStream_t stream = (cudaStream_t)stream_;
    uint32_t *ws = (uint32_t *)((uint8_t *)workspace + align_up(sizeof(SelectState), 256));
    const int vec_ok = (n % 4 == 0) && (((uintptr_t)x) % 16 == 0);
    minmax_init_kernel<<<1, 256, 0, stream>>>(ws, 1);
    minmax_f32_kernel<<<dim3(video_grid(vec_ok ? n / 4 : n), 1), 256, 0, stream>>>(x, n, ws, vec_ok);
    video_minmax_export_kernel<<<1, 32, 0, stream>>>(ws, lohi_out);
    DM_LAUNCH_CHECK("video_minmax");
    return DM_OK;
}

DM_EXPORT int dm_video_scale_f32(const float *x, long long n, const float *lohi, float *out, void *stream_) {
    using namespace dm;
    video_scale_f32_kernel<<<video_grid(n), 256, 0, (cudaStream_t)stream_>>>(x, n, lohi, out);
    DM_LAUNCH_CHECK("video_scale_f32_kernel");
    return DM_OK;
}

/* radix select over a (possibly sharded) stack: init once, then for pass = 0..3: hist (local) -> [sum the histograms over ranks:
 * int32[1024] at byte offset 32 of the workspace] -> pick.  ranks[4] are GLOBAL 0-based order-statistic ranks. */
DM_EXPORT int dm_video_select_init(void *workspace, const long long ranks[4], void *stream_) {
    using namespace dm;
    for (int i = 0; i < 4; ++i) if (ranks[i] < 0 || ranks[i] >= (1ll << 31)) { set_error("dm_video_select_init: rank out of range (stack must hold < 2^31 values)"); return DM_E_INVALID; }
    select_init_kernel<<<1, 256, 0, (cudaStream_t)stream_>>>((SelectState *)workspace, 1, (uint32_t)ranks[0], (uint32_t)ranks[1], (uint32_t)ranks[2], (uint32_t)ranks[3]);
    DM_LAUNCH_CHECK("select_init_kernel");
    return DM_OK;
}
DM_EXPORT int dm_video_select_hist(const float *x, long long n, int pass, void *workspace, void *stream_) {
    using namespace dm;
    if (n > 0) {
        int sx = (int)((n + 256 * 16 - 1) / (256 * 16));
        sx = sx < 1 ? 1 : (sx > 132 * 4 ? 132 * 4 : sx);
        select_hist_kernel<<<dim3(sx, 1), 256, 0, (cudaStream_t)stream_>>>(x, n, 0, pass, (SelectState *)workspace);
        DM_LAUNCH_CHECK("select_hist_kernel");
    }
    return DM_OK;
}
DM_EXPORT int dm_video_select_pick(void *workspace, int pass, void *stream_) {
    using namespace dm;
    select_pick_kernel<<<1, 128, 0, (cudaStream_t)stream_>>>((SelectState *)workspace, pass);
    DM_LAUNCH_CHECK("select_pick_kernel");
    return DM_OK;
}
/* np.percentile's float64 interpolation of the selected order statistics -> ab_out[2] (device doubles) */
DM_EXPORT int dm_video_select_bounds(const void *workspace, double gamma_lo, double gamma_hi, double *ab_out, void *stream_) {
    using namespace dm;
    video_bounds_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>((const SelectState *)workspace, gamma_lo, gamma_hi, ab_out);
    DM_LAUNCH_CHECK("video_bounds_kernel");
    return DM_OK;
}
DM_EXPORT int dm_video_scale_f64(const float *x, long long n, const double *ab, double *out, void *stream_) {
    using namespace dm;
    video_scale_f64_kernel<<<video_grid(n), 256, 0, (cudaStream_t)stream_>>>(x, n, ab, out);
    DM_LAUNCH_CHECK("video_scale_f64_kernel");
    return DM_OK;
}

// convert_to_i16 (src/core.py:44-50) for the float64 values of a custom depth map (src/core.py:146-174): numpy evaluates
// clip(x * 65536 + 0.0001, 0, 65535.9) in float64 and truncates
namespace dm {
__global__ void __launch_bounds__(256) convert_to_i16_f64_kernel(const double *__restrict__ x, long long n, uint16_t *__restrict__ out) {
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += nthreads) {
        double q = __dadd_rn(__dmul_rn(__ldg(x + i), 65536.0), 0.0001);
        q = fmin(fmax(q, 0.0), 65535.9);
        out[i] = (q == q) ? (uint16_t)(int)q : (uint16_t)0;
    }
}
}  // namespace dm
DM_EXPORT int dm_convert_to_i16_f64(const double *x, long long n, uint16_t *out, void *stream_) {
    using namespace dm;
    if (!x || !out || n <= 0) { set_error("dm_convert_to_i16_f64: bad arguments"); return DM_E_INVALID; }
    convert_to_i16_f64_kernel<<<video_grid(n), 256, 0, (cudaStream_t)stream_>>>(x, n, out);
    DM_LAUNCH_CHECK("convert_to_i16_f64_kernel");
    return DM_OK;
}
