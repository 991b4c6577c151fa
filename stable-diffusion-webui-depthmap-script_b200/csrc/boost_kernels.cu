// D9 — BOOST ("Boosting Monocular Depth": double estimation + patch merge), the device side of estimateboost
// (src/depthmap_generation.py:774-941, :1028-1050) and of the pix2pix merge network (pix2pix/models/networks.py:444-543,
// pix2pix/models/pix2pix4depth_model.py:96-116).  The reference runs both networks in fp32 when boost is on (:268-275), so the
// merge U-Net keeps fp32 activations and feeds the fp16 tensor core with SPLIT operands: v = hi + lo (two fp16 values, 22 bits of
// significand), A' = [a_hi | a_lo | a_hi], W' = [w_hi | w_hi | w_lo], so that one fp32-accumulating GEMM of depth 3K evaluates
// a_hi w_hi + a_lo w_hi + a_hi w_lo — everything but the 2^-22 a_lo w_lo term.
//   unet_first_cols     merge input [1024^2, 2] fp32 -> columns of the outermost 4x4 / 2 conv (K = 32, zero padded to 64)
//   unet_down_cols      LeakyReLU(0.2) + im2col of a 4x4 stride-2 pad-1 conv on fp32 NHWC: [Ho*Wo, 16 C] (ky, kx, c)
//   unet_up_cols        ReLU + gather of a ConvTranspose 4x4 stride-2 pad-1 by output parity (a, b): each output pixel (2y+a, 2x+b)
//                       sees a 2x2 input neighbourhood, [H*W, 4 (C1 + C2)] per parity, channels = cat(skip, up) without materialising it
//   unet_interleave     the four parity planes [4][H*W, N] fp32 -> NHWC [2H, 2W, C] fp32; outermost: + bias, tanh -> [2H, 2W]
//   minmax partials, merge input (min-max normalise two estimates to [-1, 1]), (t+1)/2 + min-max, degree-1 least squares of
//   the base crop on the merged patch (fp64 sums) and the blend: cubic resize of the fitted patch, Gaussian mask evaluated as the
//   outer product of a bilinearly resampled 1-D profile, updated = updated (1 - m) + merged m.
//   leres_stem_im2col_f32: the LeReS stem for a crop of a planar fp32 image (BOOST hands estimateleres float crops)
//   minmax_normalise     estimatemidasBoost's per-call (x - min) / (max - min) of the crop-size prediction, with a device flag for the
//                        constant prediction the reference cannot continue from (src/depthmap_generation.py:1212-1220)
//   quantise_crops_u8    singleestimate's ZoeDepth branch: np.uint8(crop * 255) of B same-shape crops, R and B swapped (:381, :1062-1064)
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace dm {

constexpr int BOOST_PARTIALS = 528;      // 132 SMs x 4 blocks of partial minima / maxima / sums

__device__ __forceinline__ void split_store8(const float (&v)[8], __half *hi0, __half *lo, __half *hi1, bool split) {
    uint4 uh, ul;
    __half2 *ph = reinterpret_cast<__half2 *>(&uh), *pl = reinterpret_cast<__half2 *>(&ul);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
        const float2 hf = __half22float2(h);
        ph[k] = h;
        pl[k] = __floats2half2_rn(v[2 * k] - hf.x, v[2 * k + 1] - hf.y);
    }
    *reinterpret_cast<uint4 *>(hi0) = uh;
    if (split) { *reinterpret_cast<uint4 *>(lo) = ul; *reinterpret_cast<uint4 *>(hi1) = uh; }
}

// x: [H, W, 2] fp32 (outer, inner); out: [Ho*Wo, copies*64]; no activation in front of the outermost conv
__global__ void __launch_bounds__(256) unet_first_cols_kernel(const float *__restrict__ x, int H, int W, __half *__restrict__ out, int split) {
    const int Ho = H / 2, Wo = W / 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)Ho * Wo * 8) return;
    const int part = (int)(idx & 7);            // 8 columns each: parts 0-3 = kernel row ky (4 taps x 2 channels), parts 4-7 = zero padding
    const long long pix = idx >> 3;
    const int ox = (int)(pix % Wo), oy = (int)(pix / Wo);
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (part < 4) {
        const int ky = part, iy = 2 * oy - 1 + ky;
        if (iy >= 0 && iy < H) {
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
                const int ix = 2 * ox - 1 + kx;
                if (ix >= 0 && ix < W) {
                    const float2 p = *reinterpret_cast<const float2 *>(x + ((long long)iy * W + ix) * 2);
                    v[2 * kx] = p.x; v[2 * kx + 1] = p.y;
                }
            }
        }
    }
    const int ld = split ? 192 : 64;
    __half *row = out + pix * ld + part * 8;
    split_store8(v, row, row + 64, row + 128, split != 0);
}

// LeakyReLU(0.2) is applied while gathering (every down convolution but the outermost has one in front)
__global__ void __launch_bounds__(256) unet_down_cols_kernel(const float *__restrict__ x, int H, int W, int C, __half *__restrict__ out, int split) {
    const int Ho = H / 2, Wo = W / 2, c8 = C >> 3;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)Ho * Wo * 16 * c8) return;
    const int c = (int)(idx % c8) << 3;
    long long r = idx / c8;
    const int tap = (int)(r & 15);
    const long long pix = r >> 4;
    const int ox = (int)(pix % Wo), oy = (int)(pix / Wo);
    const int iy = 2 * oy - 1 + (tap >> 2), ix = 2 * ox - 1 + (tap & 3);
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const float4 *p = reinterpret_cast<const float4 *>(x + ((long long)iy * W + ix) * C + c);
        const float4 a = __ldg(p), b = __ldg(p + 1);
        const float t[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = t[k] > 0.f ? t[k] : 0.2f * t[k];
    }
    const long long K = 16ll * C;
    __half *row = out + pix * (split ? 3 * K : K) + (long long)tap * C + c;
    split_store8(v, row, row + K, row + 2 * K, split != 0);
}

// parity (a, b): taps ty, tx in {0, 1}: input row y + dy(a, ty) with kernel row ky(a, ty):
//   a = 0: (ky 1, dy 0), (ky 3, dy -1);   a = 1: (ky 0, dy +1), (ky 2, dy 0)        (oy = 2 iy - 1 + ky)
__global__ void __launch_bounds__(256) unet_up_cols_kernel(const float *__restrict__ skip, int C1, const float *__restrict__ up, int C2, int H, int W,
                                                           __half *__restrict__ out, int split) {
    const int C = C1 + C2, c8 = C >> 3;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per = (long long)H * W * 4 * c8;
    if (idx >= 4 * per) return;
    const int par = (int)(idx / per), a = par >> 1, b = par & 1;
    long long r = idx - par * per;
    const int c = (int)(r % c8) << 3;
    r /= c8;
    const int tap = (int)(r & 3);
    const long long pix = r >> 2;
    const int x = (int)(pix % W), y = (int)(pix / W);
    const int ty = tap >> 1, tx = tap & 1;
    const int iy = y + (a == 0 ? (ty == 0 ? 0 : -1) : (ty == 0 ? 1 : 0));
    const int ix = x + (b == 0 ? (tx == 0 ? 0 : -1) : (tx == 0 ? 1 : 0));
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const float *src = c < C1 ? skip + ((long long)iy * W + ix) * C1 + c : up + ((long long)iy * W + ix) * C2 + (c - C1);
        const float4 p = __ldg(reinterpret_cast<const float4 *>(src)), q = __ldg(reinterpret_cast<const float4 *>(src) + 1);
        const float t[8] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = fmaxf(t[k], 0.f);      // relu(leaky_relu(h)) = relu(h); relu(u)
    }
    const long long K = 4ll * C, ld = split ? 3 * K : K;
    __half *row = out + ((long long)par * H * W + pix) * ld + (long long)tap * C + c;
    split_store8(v, row, row + K, row + 2 * K, split != 0);
}

// tmp: [4][H*W, N] fp32 (GEMM outputs by parity) -> out NHWC [2H, 2W, C] fp32 (C <= N)
__global__ void __launch_bounds__(256) unet_interleave_kernel(const float *__restrict__ tmp, int H, int W, int N, int C, float *__restrict__ out) {
    const int c4 = C >> 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 4ll * H * W * c4) return;
    const int c = (int)(idx % c4) << 2;
    long long r = idx / c4;
    const int ox = (int)(r % (2 * W));
    const int oy = (int)(r / (2 * W));
    const int par = ((oy & 1) << 1) | (ox & 1);
    const long long pix = (long long)(oy >> 1) * W + (ox >> 1);
    *reinterpret_cast<float4 *>(out + ((long long)oy * 2 * W + ox) * C + c) =
        __ldg(reinterpret_cast<const float4 *>(tmp + ((long long)par * H * W + pix) * N + c));
}

__global__ void __launch_bounds__(256) unet_final_kernel(const float *__restrict__ tmp, int H, int W, int N, float bias, float *__restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 4ll * H * W) return;
    const int ox = (int)(idx % (2 * W)), oy = (int)(idx / (2 * W));
    const int par = ((oy & 1) << 1) | (ox & 1);
    out[idx] = tanhf(tmp[((long long)par * H * W + (long long)(oy >> 1) * W + (ox >> 1)) * N] + bias);
}

// out[i] = gamma[i % N] * (ws[0][i] + ws[1][i] + ...): the K chunks of a split-operand GEMM, added in a FIXED order by a rounding fp32 adder
__global__ void __launch_bounds__(256) sum_chunks_kernel(const float *__restrict__ ws, int nchunks, long long mn, int N, const float *__restrict__ gamma,
                                                         float *__restrict__ out) {
    const long long i4 = ((long long)blockIdx.x * 256 + threadIdx.x) * 4;
    if (i4 >= mn) return;
    float4 acc = *reinterpret_cast<const float4 *>(ws + i4);
    for (int c = 1; c < nchunks; ++c) {
        const float4 v = *reinterpret_cast<const float4 *>(ws + (long long)c * mn + i4);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    const float4 g = *reinterpret_cast<const float4 *>(gamma + (int)(i4 % N));
    *reinterpret_cast<float4 *>(out + i4) = make_float4(acc.x * g.x, acc.y * g.y, acc.z * g.z, acc.w * g.w);
}

// The outermost transposed convolution has ONE output channel: as a GEMM it is 3.2 GB of split columns for a [.., 32]-padded result.
// Direct form in exact fp32: one thread per output pixel (2y + a, 2x + b), its four taps x (C1 + C2) input channels against the parity's
// filter slice in shared memory (broadcast reads), ReLU on load, bias + tanh.  w: [4 parities][4 taps][C1 + C2].
__global__ void __launch_bounds__(256) unet_last_kernel(const float *__restrict__ skip, int C1, const float *__restrict__ up, int C2, int H, int W,
                                                        const float *__restrict__ w, float bias, float *__restrict__ out) {
    extern __shared__ float s_w[];                      // [4][4][C]
    const int C = C1 + C2;
    for (int i = threadIdx.x; i < 16 * C; i += 256) s_w[i] = w[i];
    __syncthreads();
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= 4ll * H * W) return;
    const int ox = (int)(idx % (2 * W)), oy = (int)(idx / (2 * W));
    const int a = oy & 1, b = ox & 1, y = oy >> 1, x = ox >> 1;
    const float *wp = s_w + ((a << 1) | b) * 4 * C;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
#pragma unroll
    for (int tap = 0; tap < 4; ++tap) {
        const int ty = tap >> 1, tx = tap & 1;
        const int iy = y + (a == 0 ? (ty == 0 ? 0 : -1) : (ty == 0 ? 1 : 0));
        const int ix = x + (b == 0 ? (tx == 0 ? 0 : -1) : (tx == 0 ? 1 : 0));
        if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
        const float4 *p1 = reinterpret_cast<const float4 *>(skip + ((long long)iy * W + ix) * C1);
        const float4 *wt = reinterpret_cast<const float4 *>(wp + tap * C);
        for (int c = 0; c < C1 / 4; ++c) {
            const float4 v = __ldg(p1 + c), f = wt[c];
            acc0 = fmaf(fmaxf(v.x, 0.f), f.x, acc0); acc1 = fmaf(fmaxf(v.y, 0.f), f.y, acc1);
            acc2 = fmaf(fmaxf(v.z, 0.f), f.z, acc2); acc3 = fmaf(fmaxf(v.w, 0.f), f.w, acc3);
        }
        const float4 *p2 = reinterpret_cast<const float4 *>(up + ((long long)iy * W + ix) * C2);
        wt += C1 / 4;
        for (int c = 0; c < C2 / 4; ++c) {
            const float4 v = __ldg(p2 + c), f = wt[c];
            acc0 = fmaf(fmaxf(v.x, 0.f), f.x, acc0); acc1 = fmaf(fmaxf(v.y, 0.f), f.y, acc1);
            acc2 = fmaf(fmaxf(v.z, 0.f), f.z, acc2); acc3 = fmaf(fmaxf(v.w, 0.f), f.w, acc3);
        }
    }
    out[idx] = tanhf((acc0 + acc1) + (acc2 + acc3) + bias);
}

// The outermost convolution (2 -> 64 channels, 4x4 stride 2, no activation in front): direct fp32, one thread per (output pixel, 8 channels).
// w: [64][32] with columns (ky, kx, cin)
__global__ void __launch_bounds__(256) unet_first_kernel(const float *__restrict__ x, int H, int W, const float *__restrict__ w, float *__restrict__ out) {
    __shared__ __align__(16) float s_w[32 * 64];       // transposed to [k][channel]: the 8 channel groups of a warp read 8 distinct 32-byte segments
    for (int i = threadIdx.x; i < 64 * 32; i += 256) s_w[(i & 31) * 64 + (i >> 5)] = w[i];
    __syncthreads();
    const int Ho = H / 2, Wo = W / 2;
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)Ho * Wo * 8) return;
    const int cg = (int)(idx & 7);
    const long long pix = idx >> 3;
    const int ox = (int)(pix % Wo), oy = (int)(pix / Wo);
    float v[32];
#pragma unroll
    for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
            const int iy = 2 * oy - 1 + ky, ix = 2 * ox - 1 + kx;
            float2 p = make_float2(0.f, 0.f);
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) p = __ldg(reinterpret_cast<const float2 *>(x + ((long long)iy * W + ix) * 2));
            v[(ky * 4 + kx) * 2] = p.x; v[(ky * 4 + kx) * 2 + 1] = p.y;
        }
    float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 32; ++k) {                     // ascending k per channel: the same summation order as before
        const float4 w0 = *reinterpret_cast<const float4 *>(s_w + k * 64 + cg * 8), w1 = *reinterpret_cast<const float4 *>(s_w + k * 64 + cg * 8 + 4);
        o[0] = fmaf(v[k], w0.x, o[0]); o[1] = fmaf(v[k], w0.y, o[1]); o[2] = fmaf(v[k], w0.z, o[2]); o[3] = fmaf(v[k], w0.w, o[3]);
        o[4] = fmaf(v[k], w1.x, o[4]); o[5] = fmaf(v[k], w1.y, o[5]); o[6] = fmaf(v[k], w1.z, o[6]); o[7] = fmaf(v[k], w1.w, o[7]);
    }
    float4 *dst = reinterpret_cast<float4 *>(out + pix * 64 + cg * 8);
    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
}

// ---- reductions ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) boost_minmax_kernel(const float *__restrict__ x, long long n, float *__restrict__ partial) {
    float lo = INFINITY, hi = -INFINITY;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) { const float v = x[i]; lo = fminf(lo, v); hi = fmaxf(hi, v); }
    __shared__ float s_lo[8], s_hi[8];
    for (int o = 16; o; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < 8; ++k) { lo = fminf(lo, s_lo[k]); hi = fmaxf(hi, s_hi[k]); }
        partial[2 * blockIdx.x] = lo; partial[2 * blockIdx.x + 1] = hi;
    }
}

// every block folds the (few hundred) partials itself: no extra launch, no host round trip
__device__ __forceinline__ void fold_minmax(const float *__restrict__ partial, float &lo, float &hi) {
    __shared__ float s_l, s_h;
    if (threadIdx.x < 32) {
        float l = INFINITY, h = -INFINITY;
        for (int i = threadIdx.x; i < BOOST_PARTIALS; i += 32) { l = fminf(l, partial[2 * i]); h = fmaxf(h, partial[2 * i + 1]); }
        for (int o = 16; o; o >>= 1) { l = fminf(l, __shfl_xor_sync(0xffffffffu, l, o)); h = fmaxf(h, __shfl_xor_sync(0xffffffffu, h, o)); }
        if (threadIdx.x == 0) { s_l = l; s_h = h; }
    }
    __syncthreads();
    lo = s_l; hi = s_h;
    __syncthreads();
}

// Pix2Pix4DepthModel.set_input: each estimate min-max normalised, then * 2 - 1; real_A = cat(outer, inner)
__global__ void __launch_bounds__(256) boost_merge_input_kernel(const float *__restrict__ outer, const float *__restrict__ inner, long long n,
                                                                const float *__restrict__ p_outer, const float *__restrict__ p_inner, float *__restrict__ out) {
    float olo, ohi, ilo, ihi;
    fold_minmax(p_outer, olo, ohi);
    fold_minmax(p_inner, ilo, ihi);
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float o = (outer[i] - olo) / (ohi - olo), v = (inner[i] - ilo) / (ihi - ilo);
    *reinterpret_cast<float2 *>(out + 2 * i) = make_float2(o * 2.f - 1.f, v * 2.f - 1.f);
}

// doubleestimate's tail: m = (t + 1) / 2, then (m - min m) / (max m - min m); `normalise` = 0 stops after the first step
__global__ void __launch_bounds__(256) boost_post_kernel(const float *__restrict__ t, long long n, const float *__restrict__ partial, int normalise,
                                                         float *__restrict__ out) {
    float lo = 0.f, hi = 1.f;
    if (normalise) { fold_minmax(partial, lo, hi); lo = (lo + 1.f) / 2.f; hi = (hi + 1.f) / 2.f; }
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float m = (t[i] + 1.f) / 2.f;
    out[i] = normalise ? (m - lo) / (hi - lo) : m;
}

// estimatemidasBoost's tail: (x - min) / (max - min) in fp32; a spread of at most float64 eps writes zeros and sets *degenerate (the
// reference returns a scalar 0 there, which the following cv2.resize rejects)
__global__ void __launch_bounds__(256) boost_minmax_normalise_kernel(const float *__restrict__ x, long long n, const float *__restrict__ partial,
                                                                     float *__restrict__ out, int *__restrict__ degenerate) {
    float lo, hi;
    fold_minmax(partial, lo, hi);
    const float span = hi - lo;
    const bool flat = !((double)span > 2.220446049250313e-16);
    if (flat && blockIdx.x == 0 && threadIdx.x == 0) *degenerate = 1;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    out[i] = flat ? 0.f : (x[i] - lo) / span;
}

// np.polyfit(mapped, base, 1): sums in fp64; partial[b] = {sum x, sum y, sum xx, sum xy}
__global__ void __launch_bounds__(256) boost_fit_sums_kernel(const float *__restrict__ x, const float *__restrict__ y, long long n, double *__restrict__ partial) {
    double s[4] = {0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const double a = (double)x[i], b = (double)y[i];
        s[0] += a; s[1] += b; s[2] += a * a; s[3] += a * b;
    }
    __shared__ double sh[8][4];
    for (int k = 0; k < 4; ++k)
        for (int o = 16; o; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if ((threadIdx.x & 31) == 0)
        for (int k = 0; k < 4; ++k) sh[threadIdx.x >> 5][k] = s[k];
    __syncthreads();
    if (threadIdx.x < 4) {
        double t = 0;
        for (int w = 0; w < 8; ++w) t += sh[w][threadIdx.x];
        partial[4 * blockIdx.x + threadIdx.x] = t;
    }
}

__device__ __forceinline__ void cubic_w(float t, float (&c)[4]) {       // Keys A = -0.75 (cv2.INTER_CUBIC)
    const float A = -0.75f;
    c[0] = ((A * (t + 1.f) - 5.f * A) * (t + 1.f) + 8.f * A) * (t + 1.f) - 4.f * A;
    c[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
    c[2] = ((A + 2.f) * (1.f - t) - (A + 3.f)) * (1.f - t) * (1.f - t) + 1.f;
    c[3] = 1.f - c[0] - c[1] - c[2];
}

__device__ __forceinline__ float linear_1d(const float *__restrict__ g, int n_src, int d, float scale) {   // cv2.INTER_LINEAR along one axis
    float f = ((float)d + 0.5f) * scale - 0.5f;
    int s = (int)floorf(f);
    f -= (float)s;
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
    return g[s] * (1.f - f) + g[min(s + 1, n_src - 1)] * f;
}

// updated[y1 + y, x1 + x] = updated (1 - m) + merged m;  merged = cv2 cubic resize of (slope * mapped + intercept) to (h, w),
// m = profile_h[y] * profile_w[x] (the bilinearly resampled 3000-point Gaussian profile; the 2-D mask is its outer product)
__global__ void __launch_bounds__(256) boost_blend_kernel(const float *__restrict__ mapped, int S, const double *__restrict__ fit_partial, long long n_fit,
                                                          const float *__restrict__ profile, int n_profile, float *__restrict__ updated, int pitch, int x1,
                                                          int y1, int w, int h) {
    __shared__ double s_sum[4];
    if (threadIdx.x < 4) {
        double t = 0;
        for (int i = 0; i < BOOST_PARTIALS; ++i) t += fit_partial[4 * i + threadIdx.x];
        s_sum[threadIdx.x] = t;
    }
    __syncthreads();
    // np.polyfit(x, y, 1) as the reference calls it (:911): x and y are float32, so polyfit's rcond is len(x) * eps(float32) = 2^20 * 2^-23
    // = 0.125 — the SVD least squares on the column-normalised Vandermonde matrix [x / |x|, 1 / sqrt(n)] DROPS the second singular value
    // whenever sqrt(1 - c) <= 0.125 sqrt(1 + c), c = cos(x, 1) = sum x / (|x| sqrt n): for a merged patch whose spread is below ~25 % of
    // its mean the "degree-1 fit" is the rank-1 minimum-norm solution, not the regression line (numpy warns "poorly conditioned" and
    // goes on).  The Gram matrix of two unit columns is [[1, c], [c, 1]]: eigenvectors (1, 1) / sqrt 2 and (1, -1) / sqrt 2, eigenvalues
    // 1 + c and 1 - c, so the (truncated) pseudo-inverse is closed-form in the five sums.
    const double n = (double)n_fit, sx = s_sum[0], sy = s_sum[1], sxx = s_sum[2], sxy = s_sum[3];
    const double nx = sqrt(sxx), nn = sqrt(n);
    const double c = sx / (nx * nn), b0 = sxy / nx, b1 = sy / nn;
    const double rcond = n * 1.1920928955078125e-07;
    double c0 = (b0 + b1) / (2.0 * (1.0 + c)), c1 = c0;
    if (sqrt(1.0 - c) > rcond * sqrt(1.0 + c)) { const double t = (b0 - b1) / (2.0 * (1.0 - c)); c0 += t; c1 -= t; }
    const double slope = c0 / nx, icpt = c1 / nn;
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)w * h) return;
    const int x = (int)(idx % w), y = (int)(idx / w);
    const float scy = (float)S / (float)h, scx = (float)S / (float)w;
    float fy = scy * ((float)y + 0.5f) - 0.5f, fx = scx * ((float)x + 0.5f) - 0.5f;
    const int iy = (int)floorf(fy), ix = (int)floorf(fx);
    fy -= (float)iy; fx -= (float)ix;
    float cx[4], cy[4];
    cubic_w(fx, cx);
    cubic_w(fy, cy);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int yy = min(max(iy - 1 + j, 0), S - 1);
        float r = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) r += cx[i] * mapped[(long long)yy * S + min(max(ix - 1 + i, 0), S - 1)];
        acc += cy[j] * r;
    }
    // the cubic weights sum to one, so resizing slope * mapped + intercept equals slope * resize(mapped) + intercept
    const float merged = (float)(slope * (double)acc + icpt);
    const float m = linear_1d(profile, n_profile, y, (float)n_profile / (float)h) * linear_1d(profile, n_profile, x, (float)n_profile / (float)w);
    float *u = updated + (long long)(y1 + y) * pitch + x1 + x;
    *u = *u * (1.f - m) + merged * m;
}

// cv2.resize(INTER_CUBIC) of `planes` fp32 planes with row pitches (a crop is a pointer offset + the pitch of its parent)
__global__ void __launch_bounds__(256) boost_resize_cubic_kernel(const float *__restrict__ in, int in_pitch, long long in_plane, int Hin, int Win,
                                                                 float *__restrict__ out, int out_pitch, long long out_plane, int Hout, int Wout, int planes) {
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)planes * Hout * Wout) return;
    const int x = (int)(idx % Wout), y = (int)((idx / Wout) % Hout), pl = (int)(idx / ((long long)Wout * Hout));
    const float *img = in + pl * in_plane;
    float *dst = out + pl * out_plane + (long long)y * out_pitch + x;
    if (Hin == Hout && Win == Wout) { *dst = img[(long long)y * in_pitch + x]; return; }      // cv2.resize to the same size copies
    const float scy = (float)Hin / (float)Hout, scx = (float)Win / (float)Wout;
    float fy = scy * ((float)y + 0.5f) - 0.5f, fx = scx * ((float)x + 0.5f) - 0.5f;
    const int iy = (int)floorf(fy), ix = (int)floorf(fx);
    fy -= (float)iy; fx -= (float)ix;
    float cx[4], cy[4];
    cubic_w(fx, cx);
    cubic_w(fy, cy);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int yy = min(max(iy - 1 + j, 0), Hin - 1);
        float r = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) r += cx[i] * img[(long long)yy * in_pitch + min(max(ix - 1 + i, 0), Win - 1)];
        acc += cy[j] * r;
    }
    *dst = acc;
}

__global__ void __launch_bounds__(256) boost_u8_to_planar_kernel(const uint8_t *__restrict__ rgb, long long hw, float *__restrict__ out) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= hw) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * hw + i] = (float)((double)rgb[3 * i + c] / 255.0);
}

// ---- LeReS stem for a crop of a planar fp32 image ---------------------------------------------------------------------------
struct StemF32Params {
    const float *img;       // [3, Hi, Wi] (network channel order), values as handed to estimateleres (no / 255)
    const int *rects;       // optional [B][4] = x0, y0, w, h per batch item (device memory): B crops of the same image in one launch
    long long plane;
    int B, pitch, x0, y0, w, h, nh, nw, Ho, Wo;
    float mean[3], inv_std[3];
    __half *out;            // [Ho*Wo, 192]
};

__device__ __forceinline__ void cv_linear_coord_f(int d, float scale, int n_src, int &i0, int &i1, float &f) {
    float fx = ((float)d + 0.5f) * scale - 0.5f;
    int sx = (int)floorf(fx);
    fx -= (float)sx;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= n_src - 1) { fx = 0.f; sx = n_src - 1; }
    i0 = sx; i1 = min(sx + 1, n_src - 1); f = fx;
}

__device__ __forceinline__ void stem_flush_rows_f32(const __half *s_rows, __half *out, long long first_pix, long long total_pix) {
    const long long rows = min((long long)32, total_pix - first_pix);
    const uint4 *src = reinterpret_cast<const uint4 *>(s_rows);
    uint4 *dst = reinterpret_cast<uint4 *>(out + first_pix * 192);
    for (int i = threadIdx.x; i < (int)rows * 24; i += 256) dst[i] = src[i];
}

// rows assembled in shared memory and written with 16-byte stores (see leres_kernels.cu).  CIRCULAR: the padding wraps around the
// network input before the resize (leres_kernels.cu)
template <bool CIRCULAR>
__global__ void __launch_bounds__(256) leres_stem_im2col_f32_kernel(StemF32Params p) {
    __shared__ __align__(16) __half s_rows[32 * 192];
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total_pix = (long long)p.B * p.Ho * p.Wo;
    const int ky = (int)(idx & 7);
    const long long pix = idx >> 3;
    const bool live = pix < total_pix;
    __half *row = s_rows + (threadIdx.x >> 3) * 192;
    if (live && ky == 7) {
        for (int k = 147; k < 192; ++k) row[k] = __float2half_rn(0.f);
    } else if (live) {
        const int ox = (int)(pix % p.Wo), oy = (int)((pix / p.Wo) % p.Ho);
        if (p.rects) {
            const int4 r = __ldg(reinterpret_cast<const int4 *>(p.rects) + (int)(pix / ((long long)p.Wo * p.Ho)));
            p.x0 = r.x; p.y0 = r.y; p.w = r.z; p.h = r.w;
        }
        const bool identity = p.nh == p.h && p.nw == p.w;
        const float sy = (float)p.h / (float)p.nh, sx = (float)p.w / (float)p.nw;
        const int iy = CIRCULAR ? wrap_index(oy * 2 - 3 + ky, p.nh) : oy * 2 - 3 + ky;
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = CIRCULAR ? wrap_index(ox * 2 - 3 + kx, p.nw) : ox * 2 - 3 + kx;
            float v[3] = {0.f, 0.f, 0.f};
            if (iy >= 0 && iy < p.nh && ix >= 0 && ix < p.nw) {
                int y0 = iy, y1 = iy, x0 = ix, x1 = ix; float fy = 0.f, fx = 0.f;
                if (!identity) { cv_linear_coord_f(iy, sy, p.h, y0, y1, fy); cv_linear_coord_f(ix, sx, p.w, x0, x1, fx); }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float *pl = p.img + c * p.plane + (long long)p.y0 * p.pitch + p.x0;
                    const float a = pl[(long long)y0 * p.pitch + x0] * (1.f - fx) + pl[(long long)y0 * p.pitch + x1] * fx;
                    const float d = pl[(long long)y1 * p.pitch + x0] * (1.f - fx) + pl[(long long)y1 * p.pitch + x1] * fx;
                    v[c] = ((a * (1.f - fy) + d * fy) - p.mean[c]) * p.inv_std[c];
                }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) row[(ky * 7 + kx) * 3 + c] = __float2half_rn(v[c]);
        }
    }
    __syncthreads();
    stem_flush_rows_f32(s_rows, p.out, (long long)blockIdx.x * 32, total_pix);
}

// singleestimate's ZoeDepth branch (src/depthmap_generation.py:1062-1064) hands PIL np.uint8(img * 255) of the float64 crop: the
// product in double, truncated toward zero, the low 8 bits kept (x86-64: cubic overshoot wraps, 260.1 -> 4, -2.5 -> 254).  img is
// what get_raw_prediction made of the image (:381), R and B swapped: byte c of a pixel comes from plane 2 - c.  One thread per
// pixel; consecutive threads read consecutive floats of each plane and write consecutive bytes.
__global__ void __launch_bounds__(256) boost_quantise_crops_u8_kernel(const float *__restrict__ img, long long plane, int pitch,
                                                                       const int *__restrict__ rects, int h, int w, long long total,
                                                                       uint8_t *__restrict__ out) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int x = (int)(i % w);
    const long long by = i / w;
    const int y = (int)(by % h), b = (int)(by / h);
    const float *src = img + (long long)(rects[4 * b + 1] + y) * pitch + rects[4 * b] + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double v = (double)__ldg(src + (2 - c) * plane) * 255.0;
        out[3 * i + c] = (uint8_t)(unsigned)__double2int_rz(v);
    }
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))
#define GRID(n) (unsigned)(((n) + 255) / 256)

DM_EXPORT int dm_boost_partials(void) { return dm::BOOST_PARTIALS; }

DM_EXPORT int dm_unet_first_cols(const float *x, int H, int W, void *out, int split, void *stream_) {
    using namespace dm;
    if (!x || !out || (H & 1) || (W & 1)) { set_error("dm_unet_first_cols: bad arguments"); return DM_E_INVALID; }
    unet_first_cols_kernel<<<GRID((long long)(H / 2) * (W / 2) * 8), 256, 0, (cudaStream_t)stream_>>>(x, H, W, (__half *)out, split);
    DM_LAUNCH_CHECK("unet_first_cols_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_down_cols(const float *x, int H, int W, int C, void *out, int split, void *stream_) {
    using namespace dm;
    if (!x || !out || (H & 1) || (W & 1) || (C % 8)) { set_error("dm_unet_down_cols: bad arguments (C must be a multiple of 8)"); return DM_E_INVALID; }
    unet_down_cols_kernel<<<GRID((long long)(H / 2) * (W / 2) * 16 * (C / 8)), 256, 0, (cudaStream_t)stream_>>>(x, H, W, C, (__half *)out, split);
    DM_LAUNCH_CHECK("unet_down_cols_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_up_cols(const float *skip, int C1, const float *up, int C2, int H, int W, void *out, int split, void *stream_) {
    using namespace dm;
    if (!skip || !out || (C1 % 8) || (C2 % 8) || (C2 > 0 && !up)) { set_error("dm_unet_up_cols: bad arguments"); return DM_E_INVALID; }
    unet_up_cols_kernel<<<GRID(4ll * H * W * 4 * ((C1 + C2) / 8)), 256, 0, (cudaStream_t)stream_>>>(skip, C1, up, C2, H, W, (__half *)out, split);
    DM_LAUNCH_CHECK("unet_up_cols_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_interleave(const float *tmp, int H, int W, int N, int C, float *out, void *stream_) {
    using namespace dm;
    if (!tmp || !out || (C % 4) || C > N) { set_error("dm_unet_interleave: bad arguments"); return DM_E_INVALID; }
    unet_interleave_kernel<<<GRID(4ll * H * W * (C / 4)), 256, 0, (cudaStream_t)stream_>>>(tmp, H, W, N, C, out);
    DM_LAUNCH_CHECK("unet_interleave_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_final(const float *tmp, int H, int W, int N, float bias, float *out, void *stream_) {
    using namespace dm;
    if (!tmp || !out) { set_error("dm_unet_final: null argument"); return DM_E_INVALID; }
    unet_final_kernel<<<GRID(4ll * H * W), 256, 0, (cudaStream_t)stream_>>>(tmp, H, W, N, bias, out);
    DM_LAUNCH_CHECK("unet_final_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_last(const float *skip, int C1, const float *up, int C2, int H, int W, const float *w, float bias, float *out, void *stream_) {
    using namespace dm;
    if (!skip || !up || !w || !out || (C1 % 4) || (C2 % 4) || 16 * (C1 + C2) * 4 > 48 * 1024) { set_error("dm_unet_last: bad arguments"); return DM_E_INVALID; }
    unet_last_kernel<<<GRID(4ll * H * W), 256, 16 * (C1 + C2) * sizeof(float), (cudaStream_t)stream_>>>(skip, C1, up, C2, H, W, w, bias, out);
    DM_LAUNCH_CHECK("unet_last_kernel");
    return DM_OK;
}

DM_EXPORT int dm_unet_first(const float *x, int H, int W, const float *w, float *out, void *stream_) {
    using namespace dm;
    if (!x || !w || !out || (H & 1) || (W & 1)) { set_error("dm_unet_first: bad arguments"); return DM_E_INVALID; }
    unet_first_kernel<<<GRID((long long)(H / 2) * (W / 2) * 8), 256, 0, (cudaStream_t)stream_>>>(x, H, W, w, out);
    DM_LAUNCH_CHECK("unet_first_kernel");
    return DM_OK;
}

DM_EXPORT int dm_sum_chunks_f32(const float *ws, int nchunks, long long mn, int N, const float *gamma, float *out, void *stream_) {
    using namespace dm;
    if (!ws || !gamma || !out || nchunks < 1 || (N % 4) || (mn % N)) { set_error("dm_sum_chunks_f32: bad arguments"); return DM_E_INVALID; }
    sum_chunks_kernel<<<GRID(mn / 4), 256, 0, (cudaStream_t)stream_>>>(ws, nchunks, mn, N, gamma, out);
    DM_LAUNCH_CHECK("sum_chunks_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_minmax(const float *x, long long n, float *partial, void *stream_) {
    using namespace dm;
    if (!x || !partial || n <= 0) { set_error("dm_boost_minmax: bad arguments"); return DM_E_INVALID; }
    boost_minmax_kernel<<<BOOST_PARTIALS, 256, 0, (cudaStream_t)stream_>>>(x, n, partial);
    DM_LAUNCH_CHECK("boost_minmax_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_merge_input(const float *outer, const float *inner, long long n, const float *p_outer, const float *p_inner, float *out, void *stream_) {
    using namespace dm;
    if (!outer || !inner || !p_outer || !p_inner || !out) { set_error("dm_boost_merge_input: null argument"); return DM_E_INVALID; }
    boost_merge_input_kernel<<<GRID(n), 256, 0, (cudaStream_t)stream_>>>(outer, inner, n, p_outer, p_inner, out);
    DM_LAUNCH_CHECK("boost_merge_input_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_post(const float *t, long long n, const float *partial, int normalise, float *out, void *stream_) {
    using namespace dm;
    if (!t || !out || (normalise && !partial)) { set_error("dm_boost_post: null argument"); return DM_E_INVALID; }
    boost_post_kernel<<<GRID(n), 256, 0, (cudaStream_t)stream_>>>(t, n, partial, normalise, out);
    DM_LAUNCH_CHECK("boost_post_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_minmax_normalise(const float *x, long long n, const float *partial, float *out, int *degenerate, void *stream_) {
    using namespace dm;
    if (!x || !partial || !out || !degenerate || n <= 0) { set_error("dm_boost_minmax_normalise: bad arguments"); return DM_E_INVALID; }
    boost_minmax_normalise_kernel<<<GRID(n), 256, 0, (cudaStream_t)stream_>>>(x, n, partial, out, degenerate);
    DM_LAUNCH_CHECK("boost_minmax_normalise_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_fit_sums(const float *x, const float *y, long long n, double *partial, void *stream_) {
    using namespace dm;
    if (!x || !y || !partial) { set_error("dm_boost_fit_sums: null argument"); return DM_E_INVALID; }
    boost_fit_sums_kernel<<<BOOST_PARTIALS, 256, 0, (cudaStream_t)stream_>>>(x, y, n, partial);
    DM_LAUNCH_CHECK("boost_fit_sums_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_blend(const float *mapped, int S, const double *fit_partial, const float *profile, int n_profile, float *updated, int pitch, int x1,
                             int y1, int w, int h, void *stream_) {
    using namespace dm;
    if (!mapped || !fit_partial || !profile || !updated || w <= 0 || h <= 0) { set_error("dm_boost_blend: bad arguments"); return DM_E_INVALID; }
    boost_blend_kernel<<<GRID((long long)w * h), 256, 0, (cudaStream_t)stream_>>>(mapped, S, fit_partial, (long long)S * S, profile, n_profile, updated, pitch,
                                                                                 x1, y1, w, h);
    DM_LAUNCH_CHECK("boost_blend_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_resize_cubic(const float *in, int in_pitch, long long in_plane, int Hin, int Win, float *out, int out_pitch, long long out_plane,
                                    int Hout, int Wout, int planes, void *stream_) {
    using namespace dm;
    if (!in || !out || Hin <= 0 || Win <= 0 || Hout <= 0 || Wout <= 0 || planes <= 0) { set_error("dm_boost_resize_cubic: bad arguments"); return DM_E_INVALID; }
    boost_resize_cubic_kernel<<<GRID((long long)planes * Hout * Wout), 256, 0, (cudaStream_t)stream_>>>(in, in_pitch, in_plane, Hin, Win, out, out_pitch,
                                                                                                        out_plane, Hout, Wout, planes);
    DM_LAUNCH_CHECK("boost_resize_cubic_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_u8_to_planar(const uint8_t *rgb, int H, int W, float *out, void *stream_) {
    using namespace dm;
    if (!rgb || !out) { set_error("dm_boost_u8_to_planar: null argument"); return DM_E_INVALID; }
    boost_u8_to_planar_kernel<<<GRID((long long)H * W), 256, 0, (cudaStream_t)stream_>>>(rgb, (long long)H * W, out);
    DM_LAUNCH_CHECK("boost_u8_to_planar_kernel");
    return DM_OK;
}

DM_EXPORT int dm_boost_quantise_crops_u8(const float *img, int Hi, int Wi, const int *rects_dev, int B, int h, int w, uint8_t *out, void *stream_) {
    using namespace dm;
    if (!img || !rects_dev || !out || B <= 0 || h <= 0 || w <= 0 || h > Hi || w > Wi) {
        set_error("dm_boost_quantise_crops_u8: bad arguments");
        return DM_E_INVALID;
    }
    const long long total = (long long)B * h * w;
    boost_quantise_crops_u8_kernel<<<GRID(total), 256, 0, (cudaStream_t)stream_>>>(img, (long long)Hi * Wi, Wi, rects_dev, h, w, total, out);
    DM_LAUNCH_CHECK("boost_quantise_crops_u8_kernel");
    return DM_OK;
}

template <bool CIRCULAR>
static int leres_stem_im2col_f32(const char *who, const float *img, int Hi, int Wi, int x0, int y0, int w, int h, int net_h, int net_w,
                                 const float *mean_host, const float *std_host, void *out, void *stream_) {
    using namespace dm;
    if (!img || !out || x0 < 0 || y0 < 0 || w <= 0 || h <= 0 || x0 + w > Wi || y0 + h > Hi) { set_error("%s: crop outside the image", who); return DM_E_INVALID; }
    StemF32Params p;
    p.rects = nullptr; p.B = 1;
    p.img = img; p.plane = (long long)Hi * Wi; p.pitch = Wi; p.x0 = x0; p.y0 = y0; p.w = w; p.h = h; p.nh = net_h; p.nw = net_w;
    p.Ho = (net_h + 6 - 7) / 2 + 1; p.Wo = (net_w + 6 - 7) / 2 + 1;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; }
    p.out = (__half *)out;
    leres_stem_im2col_f32_kernel<CIRCULAR><<<GRID((long long)p.Ho * p.Wo * 8), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("leres_stem_im2col_f32_kernel");
    return DM_OK;
}

DM_EXPORT int dm_leres_stem_im2col_f32(const float *img, int Hi, int Wi, int x0, int y0, int w, int h, int net_h, int net_w, const float *mean_host,
                                       const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_f32<false>("dm_leres_stem_im2col_f32", img, Hi, Wi, x0, y0, w, h, net_h, net_w, mean_host, std_host, out, stream_);
}

DM_EXPORT int dm_leres_stem_im2col_f32_circular(const float *img, int Hi, int Wi, int x0, int y0, int w, int h, int net_h, int net_w,
                                                const float *mean_host, const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_f32<true>("dm_leres_stem_im2col_f32_circular", img, Hi, Wi, x0, y0, w, h, net_h, net_w, mean_host, std_host, out, stream_);
}

/* B crops of the same planar image in one launch; rects: device int32 [B][4] = x0, y0, w, h (validated by the caller) */
template <bool CIRCULAR>
static int leres_stem_im2col_f32_batch(const char *who, const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w,
                                       const float *mean_host, const float *std_host, void *out, void *stream_) {
    using namespace dm;
    if (!img || !out || !rects_dev || B <= 0) { set_error("%s: bad arguments", who); return DM_E_INVALID; }
    StemF32Params p;
    p.rects = rects_dev; p.B = B;
    p.img = img; p.plane = (long long)Hi * Wi; p.pitch = Wi; p.x0 = 0; p.y0 = 0; p.w = Wi; p.h = Hi; p.nh = net_h; p.nw = net_w;
    p.Ho = (net_h + 6 - 7) / 2 + 1; p.Wo = (net_w + 6 - 7) / 2 + 1;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; }
    p.out = (__half *)out;
    leres_stem_im2col_f32_kernel<CIRCULAR><<<GRID((long long)B * p.Ho * p.Wo * 8), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("leres_stem_im2col_f32_kernel");
    return DM_OK;
}

DM_EXPORT int dm_leres_stem_im2col_f32_batch(const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w, const float *mean_host,
                                             const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_f32_batch<false>("dm_leres_stem_im2col_f32_batch", img, Hi, Wi, rects_dev, B, net_h, net_w, mean_host, std_host, out, stream_);
}

DM_EXPORT int dm_leres_stem_im2col_f32_batch_circular(const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w,
                                                      const float *mean_host, const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_f32_batch<true>("dm_leres_stem_im2col_f32_batch_circular", img, Hi, Wi, rects_dev, B, net_h, net_w, mean_host, std_host, out,
                                             stream_);
}
