// D7 — ZoeDepth-NK: everything around the DPT-BEiT core that the reference's DepthModel / ZoeDepthNK adds
// (dzoedepth/models/depth_model.py:57-152, zoedepth_nk/zoedepth_nk_v1.py:159-243, layers/attractor.py:127-208,
// layers/dist_layers.py:29-121, layers/patch_transformer.py:29-92, base_models/midas.py:175-186).
// The 1x1 convolutions of the head run on the wgmma GEMM (NHWC activations = row-major [pixels, channels]); the
// kernels here are the bandwidth-side pieces, fp32 math:
//   zoe_preprocess_patchify  ToTensor -> reflect pad -> (flip) -> bilinear align_corners=True to the net size -> (x-.5)/.5
//                            -> fp16 patch matrix; forward 2b is image b, forward 2b+1 its horizontal flip (TTA)
//   layernorm_post           post-norm transformer layer of the router: x = LN(x) in place (fp32) + fp16 copy
//   attention_small          router self-attention (4 heads x 32 dims, 257 tokens), SIMT
//   select_softplus          seed bin centres of the routed head: softplus(seed[:, head*64 : head*64+64])
//   resize_add_nhwc          x = b_emb + bilinear(prev_b_embedding)            (attractor.py:173-177)
//   attractor                b_new = b + mean_i inv_attractor(A_i - b), b = bilinear(b_prev)   (attractor.py:178-208)
//   clb_final                ConditionalLogBinomial + sum(p * bin centres) per output pixel of the routed head, with the
//                            1x1 conv on cat(out_conv, bilinear(b_emb)) split by linearity into W_o . out_conv (here) +
//                            bilinear(W_e . b_emb) (a GEMM at a quarter of the pixels)
//   tta_combine              bicubic (align_corners=False) back to the padded size, crop, average with the un-flipped
//                            flipped prediction
// The router decision is taken per forward on the device (argmax of the two logits): no host synchronisation
// (the reference calls .item(), zoedepth_nk_v1.py:194-195) and no cross-image vote (SURVEY §8e).
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace dm {

__device__ __forceinline__ void cubic_coeffs_z(float x, float *c) {
    const float A = -0.75f;
    c[0] = ((A * (x + 1.f) - 5.f * A) * (x + 1.f) + 8.f * A) * (x + 1.f) - 4.f * A;
    c[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
    c[2] = ((A + 2.f) * (1.f - x) - (A + 3.f)) * (1.f - x) * (1.f - x) + 1.f;
    c[3] = 1.f - c[0] - c[1] - c[2];
}
__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }   // F.softplus defaults
__device__ __forceinline__ int route_of(const float *logits, int ld, int f) { return logits[(size_t)f * ld + 1] > logits[(size_t)f * ld] ? 1 : 0; }

// ---------------------------------------------------------------------------------------------------------------
struct ZoePre {
    const uint8_t *rgb;
    int B, H, W, pad_h, pad_w, nh, nw, patch, gh, gw, kpad;
    __half *out;
};

__global__ void __launch_bounds__(256) zoe_preprocess_patchify_kernel(ZoePre p) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)2 * p.B * p.nh * p.nw;
    if (idx >= total) return;
    const int x = (int)(idx % p.nw);
    const int y = (int)((idx / p.nw) % p.nh);
    const int f = (int)(idx / ((long long)p.nw * p.nh));
    const int b = f >> 1, flip = f & 1;
    const int Hp = p.H + 2 * p.pad_h, Wp = p.W + 2 * p.pad_w;
    const uint8_t *img = p.rgb + (long long)b * p.H * p.W * 3;
    // F.interpolate(bilinear, align_corners=True) over the padded (and flipped) image
    const float sy = p.nh > 1 ? (float)(Hp - 1) / (float)(p.nh - 1) : 0.f;
    const float sx = p.nw > 1 ? (float)(Wp - 1) / (float)(p.nw - 1) : 0.f;
    const float fy = sy * (float)y, fx = sx * (float)x;
    const int y0 = min((int)fy, Hp - 1), x0 = min((int)fx, Wp - 1);
    const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    auto src = [&](int yy, int xx, float *v) {
        if (flip) xx = Wp - 1 - xx;
        int sy_ = yy - p.pad_h, sx_ = xx - p.pad_w;           // F.pad(mode="reflect"): edge not repeated
        sy_ = sy_ < 0 ? -sy_ : (sy_ >= p.H ? 2 * (p.H - 1) - sy_ : sy_);
        sx_ = sx_ < 0 ? -sx_ : (sx_ >= p.W ? 2 * (p.W - 1) - sx_ : sx_);
        const uint8_t *px = img + ((long long)sy_ * p.W + sx_) * 3;
        v[0] = (float)px[0] / 255.0f; v[1] = (float)px[1] / 255.0f; v[2] = (float)px[2] / 255.0f;   // transforms.ToTensor
    };
    float v00[3], v01[3], v10[3], v11[3];
    src(y0, x0, v00); src(y0, x1, v01); src(y1, x0, v10); src(y1, x1, v11);
    const int py = y / p.patch, ky = y % p.patch, pxi = x / p.patch, kx = x % p.patch;
    __half *row = p.out + ((long long)(f * p.gh + py) * p.gw + pxi) * p.kpad;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float r = hy * (hx * v00[c] + lx * v01[c]) + ly * (hx * v10[c] + lx * v11[c]);
        row[(c * p.patch + ky) * p.patch + kx] = __float2half_rn((r - 0.5f) / 0.5f);
    }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm_post_kernel(float *__restrict__ x, long long rows, const float *__restrict__ gamma,
                                                             const float *__restrict__ beta, float eps, __half *__restrict__ out) {
    // C = 128: one warp per row, one float4 per lane
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    float4 v = reinterpret_cast<const float4 *>(x + row * 128)[lane];
    float s = (v.x + v.y) + (v.z + v.w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / 128.f;
    const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
    float q = (a * a + b * b) + (c * c + d * d);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / 128.f + eps);
    const float4 g = reinterpret_cast<const float4 *>(gamma)[lane], bt = reinterpret_cast<const float4 *>(beta)[lane];
    v = make_float4(a * rstd * g.x + bt.x, b * rstd * g.y + bt.y, c * rstd * g.z + bt.z, d * rstd * g.w + bt.w);
    reinterpret_cast<float4 *>(x + row * 128)[lane] = v;
    const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t *>(&h0);
    u.y = *reinterpret_cast<const uint32_t *>(&h1);
    reinterpret_cast<uint2 *>(out + row * 128)[lane] = u;
}

// router attention: qkv fp16 [F*S, 3*E] (q | k | v, head h at columns h*32), out fp16 [F*S, E]; grid (F, heads)
constexpr int RA_HD = 32, RA_PITCH = 33;
__global__ void __launch_bounds__(256) attention_small_kernel(const __half *__restrict__ qkv, int S, int E, float scale, __half *__restrict__ out) {
    extern __shared__ float ra_smem[];
    float *sk = ra_smem, *sv = sk + (size_t)S * RA_PITCH, *sp = sv + (size_t)S * RA_PITCH;   // sp: [8 warps][S]
    const int f = blockIdx.x, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const __half *base = qkv + (size_t)f * S * 3 * E + h * RA_HD;
    for (int i = threadIdx.x; i < S * RA_HD; i += 256) {
        const int t = i >> 5, d = i & 31;
        sk[t * RA_PITCH + d] = __half2float(base[(size_t)t * 3 * E + E + d]);
        sv[t * RA_PITCH + d] = __half2float(base[(size_t)t * 3 * E + 2 * E + d]);
    }
    __syncthreads();
    float *pw = sp + (size_t)warp * S;
    const int rows_per = (S + gridDim.z - 1) / gridDim.z, t_beg = blockIdx.z * rows_per, t_end = min(S, t_beg + rows_per);
    for (int t = t_beg + warp; t < t_end; t += 8) {
        const float qd = __half2float(base[(size_t)t * 3 * E + lane]) * scale;
        float mx = -INFINITY;
        for (int j0 = 0; j0 < S; j0 += 32) {                 // uniform trip count: the shuffles need every lane
            const int j = j0 + lane;
            const float *kr = sk + (size_t)min(j, S - 1) * RA_PITCH;
            float s = 0.f;
#pragma unroll
            for (int d = 0; d < RA_HD; ++d) s = fmaf(__shfl_sync(0xffffffffu, qd, d), kr[d], s);
            if (j < S) { pw[j] = s; mx = fmaxf(mx, s); }
        }
        __syncwarp();
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
        for (int j = lane; j < S; j += 32) { const float e = __expf(pw[j] - mx); pw[j] = e; sum += e; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        __syncwarp();
        float acc = 0.f;                                    // lane = output dim
        for (int j = 0; j < S; ++j) acc = fmaf(pw[j], sv[j * RA_PITCH + lane], acc);
        out[((size_t)f * S + t) * E + h * RA_HD + lane] = __float2half_rn(acc / sum);
        __syncwarp();
    }
}

__global__ void __launch_bounds__(256) cast_f32_f16_kernel(const float *__restrict__ x, long long n4, __half *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = reinterpret_cast<const float4 *>(x)[i];
    const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t *>(&h0);
    u.y = *reinterpret_cast<const uint32_t *>(&h1);
    reinterpret_cast<uint2 *>(out)[i] = u;
}

__global__ void __launch_bounds__(256) select_softplus_kernel(const float *__restrict__ seed, int ld, const float *__restrict__ logits, int lld,
                                                              long long rows, int rows_per_fwd, float *__restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * 64) return;
    const long long r = idx >> 6;
    const int k = (int)(idx & 63);
    const int head = route_of(logits, lld, (int)(r / rows_per_fwd));
    out[idx] = softplus_f(seed[r * ld + head * 64 + k]);
}

// out = a + bilinear_align_corners(b), NHWC fp16, 8 channels per thread; grid (ceil(W*C/8/256), H, B)
__global__ void __launch_bounds__(256) resize_add_nhwc_kernel(const __half *__restrict__ a, const __half *__restrict__ bsm, int Hs, int Ws, int C,
                                                              __half *__restrict__ out, int H, int W, float sy, float sx) {
    const int c8 = C >> 3;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= W * c8) return;
    const int x = t / c8;
    const int c = (t - x * c8) << 3;
    const int y = blockIdx.y, b = blockIdx.z;
    const float fy = sy * (float)y, fx = sx * (float)x;
    const int y0 = min((int)fy, Hs - 1), x0 = min((int)fx, Ws - 1);
    const int y1 = min(y0 + 1, Hs - 1), x1 = min(x0 + 1, Ws - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const __half *base = bsm + (size_t)b * Hs * Ws * C + c;
    const uint4 u00 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y0 * Ws + x0) * C));
    const uint4 u01 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y0 * Ws + x1) * C));
    const uint4 u10 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y1 * Ws + x0) * C));
    const uint4 u11 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y1 * Ws + x1) * C));
    const size_t o_off = ((size_t)(b * H + y) * W + x) * C + c;
    const uint4 ua = __ldg(reinterpret_cast<const uint4 *>(a + o_off));
    const __half2 *p00 = reinterpret_cast<const __half2 *>(&u00), *p01 = reinterpret_cast<const __half2 *>(&u01);
    const __half2 *p10 = reinterpret_cast<const __half2 *>(&u10), *p11 = reinterpret_cast<const __half2 *>(&u11);
    const __half2 *pa = reinterpret_cast<const __half2 *>(&ua);
    uint4 o;
    __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 f00 = __half22float2(p00[k]), f01 = __half22float2(p01[k]), f10 = __half22float2(p10[k]), f11 = __half22float2(p11[k]);
        const float2 fa = __half22float2(pa[k]);
        oh[k] = __floats2half2_rn(fa.x + (hy * (hx * f00.x + lx * f01.x) + ly * (hx * f10.x + lx * f11.x)),
                                  fa.y + (hy * (hx * f00.y + lx * f01.y) + ly * (hx * f10.y + lx * f11.y)));
    }
    *reinterpret_cast<uint4 *>(out + o_off) = o;
}

// b_new[f, y, x, k] = b + (1/16) * sum_i dx_i / (1 + 300 dx_i^2), dx_i = softplus(A[f, y, x, head*32 + i]) - b,
// b = bilinear_align_corners(b_prev)[k].  One thread per (pixel, bin); the 16 attractors of a pixel are broadcast by shuffle.
__global__ void __launch_bounds__(256) attractor_kernel(const float *__restrict__ A, int lda, const float *__restrict__ logits, int lld,
                                                        const float *__restrict__ bprev, int Hp, int Wp, int H, int W, float sy, float sx,
                                                        float *__restrict__ bout) {
    const int y = blockIdx.y, f = blockIdx.z;
    const int t = blockIdx.x * 256 + threadIdx.x;       // (x, bin): 64 bins per pixel -> half a warp per pixel
    const int x = t >> 6, k = t & 63;
    const int lane = threadIdx.x & 31;
    const bool ok = x < W;
    const int xc = ok ? x : W - 1;
    const int head = route_of(logits, lld, f);
    const float fy = sy * (float)y, fx = sx * (float)xc;
    const int y0 = min((int)fy, Hp - 1), x0 = min((int)fx, Wp - 1);
    const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const float *bp = bprev + (size_t)f * Hp * Wp * 64 + k;
    const float b = hy * (hx * bp[(size_t)(y0 * Wp + x0) * 64] + lx * bp[(size_t)(y0 * Wp + x1) * 64]) +
                    ly * (hx * bp[(size_t)(y1 * Wp + x0) * 64] + lx * bp[(size_t)(y1 * Wp + x1) * 64]);
    // lanes 0..15 of the warp fetch the 16 attractor points of this warp's pixel (a warp covers 32 bins of ONE pixel)
    const float *arow = A + ((size_t)(f * H + y) * W + xc) * lda + head * 32;
    const float a_mine = softplus_f(arow[lane & 15]);
    float delta = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const float dx = __shfl_sync(0xffffffffu, a_mine, i) - b;
        delta += __fdividef(dx, 1.f + 300.f * (dx * dx));      // 2 ulp; the head's bar is a tolerance, and this is 16 divisions per thread
    }
    if (ok) bout[((size_t)(f * H + y) * W + x) * 64 + k] = b + delta / 16.f;
}

// ---------------------------------------------------------------------------------------------------------------
struct ClbParams {
    const __half *o32; int ldo;          // [F, nh, nw, ldo] relu'd out_conv activation, channels 0..31
    const float *ze; int ldz;            // [F, h3, w3, ldz]: W_e . b_emb, nyu at columns 0..39, kitti at 64..103
    const float *bc;                     // [F, h3, w3, 64] bin centres of the routed head
    const float *logits; int lld;
    const float *wo;                     // [2][32][40]  (input channel major)
    const float *b0;                     // [2][40]
    const float *w2;                     // [2][4][40]
    const float *b2;                     // [2][4]
    int F, nh, nw, h3, w3;
    float sy, sx, min_temp, max_temp;
    float *out;                          // [F, nh, nw]
};

__device__ __forceinline__ float log_binom_f(float n, float k) {   // dist_layers.py:29-33 (eps = 1e-7 added to n and k)
    n += 1e-7f; k += 1e-7f;
    return n * logf(n) - k * logf(k) - (n - k) * logf(n - k + 1e-7f);
}

// One THREAD per output pixel (the first version spent a warp per pixel: ~900 warp-instructions per pixel in shuffles, reductions
// and scalar work replicated 32 times; this form needs ~110).  The weights sit in shared memory and are read as broadcasts; a
// thread's loads are whole contiguous vectors (64 B of out_conv, 160 B per neighbour of ze, 256 B per neighbour of the bin centres)
// and neighbouring threads share their bilinear neighbours in L1.
__global__ void __launch_bounds__(128) clb_final_kernel(ClbParams p) {
    __shared__ float s_wo[32 * 40], s_b0[40], s_w2[4 * 40], s_b2[4], s_lb[64];
    const int f = blockIdx.z;
    const int head = route_of(p.logits, p.lld, f);
    for (int i = threadIdx.x; i < 32 * 40; i += 128) s_wo[i] = p.wo[head * 32 * 40 + i];
    for (int i = threadIdx.x; i < 4 * 40; i += 128) s_w2[i] = p.w2[head * 4 * 40 + i];
    if (threadIdx.x < 40) s_b0[threadIdx.x] = p.b0[head * 40 + threadIdx.x];
    if (threadIdx.x < 4) s_b2[threadIdx.x] = p.b2[head * 4 + threadIdx.x];
    if (threadIdx.x < 64) s_lb[threadIdx.x] = log_binom_f(63.f, (float)threadIdx.x);
    __syncthreads();
    const int y = blockIdx.y, x = blockIdx.x * 128 + threadIdx.x;
    if (x >= p.nw) return;
    const float fy = p.sy * (float)y, fx = p.sx * (float)x;
    const int y0 = min((int)fy, p.h3 - 1), y1 = min(y0 + 1, p.h3 - 1), x0 = min((int)fx, p.w3 - 1), x1 = min(x0 + 1, p.w3 - 1);
    const float ly = fy - (float)y0, hy = 1.f - ly, lx = fx - (float)x0, hx = 1.f - lx;
    const size_t i00 = ((size_t)f * p.h3 + y0) * p.w3 + x0, i01 = ((size_t)f * p.h3 + y0) * p.w3 + x1;
    const size_t i10 = ((size_t)f * p.h3 + y1) * p.w3 + x0, i11 = ((size_t)f * p.h3 + y1) * p.w3 + x1;
    // pre-activation of mlp.0 = b0 + W_o . out_conv + bilinear(W_e . b_emb)
    float pre[40];
    {
        const float4 *z00 = reinterpret_cast<const float4 *>(p.ze + i00 * p.ldz + head * 64), *z01 = reinterpret_cast<const float4 *>(p.ze + i01 * p.ldz + head * 64);
        const float4 *z10 = reinterpret_cast<const float4 *>(p.ze + i10 * p.ldz + head * 64), *z11 = reinterpret_cast<const float4 *>(p.ze + i11 * p.ldz + head * 64);
#pragma unroll
        for (int k = 0; k < 10; ++k) {
            const float4 a = __ldg(z00 + k), b = __ldg(z01 + k), c = __ldg(z10 + k), d = __ldg(z11 + k);
            pre[4 * k + 0] = s_b0[4 * k + 0] + (hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x));
            pre[4 * k + 1] = s_b0[4 * k + 1] + (hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y));
            pre[4 * k + 2] = s_b0[4 * k + 2] + (hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z));
            pre[4 * k + 3] = s_b0[4 * k + 3] + (hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w));
        }
    }
    {
        const uint4 *op = reinterpret_cast<const uint4 *>(p.o32 + (((size_t)f * p.nh + y) * p.nw + x) * p.ldo);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint4 u = __ldg(op + q);
            const __half2 *h2 = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 o2 = __half22float2(h2[e]);
                const float *w0 = s_wo + (q * 8 + 2 * e) * 40, *w1 = w0 + 40;
#pragma unroll
                for (int k = 0; k < 40; ++k) pre[k] = fmaf(w1[k], o2.y, fmaf(w0[k], o2.x, pre[k]));
            }
        }
    }
    float pt[4] = {s_b2[0], s_b2[1], s_b2[2], s_b2[3]};
#pragma unroll
    for (int k = 0; k < 40; ++k) {
        const float g = 0.5f * pre[k] * (1.f + erff(pre[k] * 0.70710678118654752f));                 // nn.GELU (erf form)
#pragma unroll
        for (int j = 0; j < 4; ++j) pt[j] = fmaf(s_w2[j * 40 + k], g, pt[j]);
    }
    const float pa = softplus_f(pt[0]) + 1e-4f, pb = softplus_f(pt[1]) + 1e-4f, ta = softplus_f(pt[2]) + 1e-4f, tb = softplus_f(pt[3]) + 1e-4f;
    const float prob = pa / (pa + pb);
    const float temp = (p.max_temp - p.min_temp) * (ta / (ta + tb)) + p.min_temp;
    const float lp = logf(fminf(fmaxf(prob, 1e-4f), 1.f)), lq = logf(fminf(fmaxf(1.f - prob, 1e-4f), 1.f));
    // softmax over the 64 bins of y_k / temp and the expectation of the (bilinearly up-sampled) bin centres; y_k is concave in k,
    // its maximum is found in a first pass without touching memory
    const float inv_t = 1.f / temp;
    float mx = -INFINITY;
#pragma unroll 8
    for (int k = 0; k < 64; ++k) mx = fmaxf(mx, (s_lb[k] + (float)k * lp + (float)(63 - k) * lq) * inv_t);
    const float4 *c00 = reinterpret_cast<const float4 *>(p.bc + i00 * 64), *c01 = reinterpret_cast<const float4 *>(p.bc + i01 * 64);
    const float4 *c10 = reinterpret_cast<const float4 *>(p.bc + i10 * 64), *c11 = reinterpret_cast<const float4 *>(p.bc + i11 * 64);
    float den = 0.f, num = 0.f;
#pragma unroll 4
    for (int k4 = 0; k4 < 16; ++k4) {
        const float4 a = __ldg(c00 + k4), b = __ldg(c01 + k4), c = __ldg(c10 + k4), d = __ldg(c11 + k4);
        const float bcv[4] = {hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x), hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y),
                              hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z), hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w)};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 4 * k4 + e;
            const float ek = expf((s_lb[k] + (float)k * lp + (float)(63 - k) * lq) * inv_t - mx);
            den += ek;
            num = fmaf(ek, bcv[e], num);
        }
    }
    p.out[((size_t)f * p.nh + y) * p.nw + x] = num / den;
}

// out[b, y, x] = 0.5 * (up(d[2b])[y + pad_h, x + pad_w] + up(d[2b+1])[y + pad_h, Wp - 1 - (x + pad_w)]), up = bicubic
// align_corners=False from (nh, nw) to the padded size (Hp, Wp); identity when the sizes agree (depth_model.py:88-89)
__global__ void __launch_bounds__(256) tta_combine_kernel(const float *__restrict__ d, int B, int nh, int nw, int Hp, int Wp, int pad_h, int pad_w,
                                                          int H, int W, float *__restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * H * W;
    if (idx >= total) return;
    const int x = (int)(idx % W);
    const int y = (int)((idx / W) % H);
    const int b = (int)(idx / ((long long)W * H));
    const bool same = (nh == Hp && nw == Wp);
    const float sy = (float)nh / (float)Hp, sx = (float)nw / (float)Wp;
    auto sample = [&](const float *img, int yy, int xx) {
        if (same) return img[(long long)yy * nw + xx];
        float fy = sy * ((float)yy + 0.5f) - 0.5f, fx = sx * ((float)xx + 0.5f) - 0.5f;
        const int iy = (int)floorf(fy), ix = (int)floorf(fx);
        fy -= (float)iy; fx -= (float)ix;
        float cx[4], cy[4];
        cubic_coeffs_z(fx, cx);
        cubic_coeffs_z(fy, cy);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yr = min(max(iy - 1 + j, 0), nh - 1);
            float r = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) r += cx[i] * img[(long long)yr * nw + min(max(ix - 1 + i, 0), nw - 1)];
            acc += cy[j] * r;
        }
        return acc;
    };
    const float a = sample(d + (long long)(2 * b) * nh * nw, y + pad_h, x + pad_w);
    const float c = sample(d + (long long)(2 * b + 1) * nh * nw, y + pad_h, Wp - 1 - (x + pad_w));
    out[idx] = (a + c) / 2.f;
}

// ---------------------------------------------------------------------------------------------------------------
// Single-head ZoeDepth (ZoeDepth-N, model type 7: softplus bins; ZoeDepth-K, model type 8: "normed" bins), the head of
// dzoedepth/models/zoedepth/zoedepth_v1.py:124-192.  No router: the kernels below have no head index.

// seed bin centres, one warp per row of 64 (two bins per lane).  softplus: SeedBinRegressorUnnormed, c = softplus(s).
// normed: SeedBinRegressor (localbins_layers.py:52-68), B = relu(s) + 1e-3, widths = (max-min) B / sum B, edges = cumsum of
// [min, widths], c = edge midpoints; then b_prev = (c - min) / (max - min) (zoedepth_v1.py:155-157).
__global__ void __launch_bounds__(256) seed_bins_kernel(const float *__restrict__ seed, int ld, long long rows, int normed, float dmin,
                                                        float dmax, float *__restrict__ out) {
    const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;                               // whole warps leave together
    const float2 s = *reinterpret_cast<const float2 *>(seed + r * ld + 2 * lane);
    float2 o;
    if (!normed) {
        o = make_float2(softplus_f(s.x), softplus_f(s.y));
    } else {
        const float b0 = fmaxf(s.x, 0.f) + 1e-3f, b1 = fmaxf(s.y, 0.f) + 1e-3f;
        float tot = b0 + b1;
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, m);
        const float rng = dmax - dmin;
        const float w0 = rng * (b0 / tot), w1 = rng * (b1 / tot);
        float inc = w0 + w1;                             // inclusive prefix over lanes of the pair sums
#pragma unroll
        for (int m = 1; m < 32; m <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, inc, m);
            if (lane >= m) inc += t;
        }
        const float e0 = dmin + (inc - (w0 + w1));       // edge 2*lane
        const float e1 = e0 + w0, e2 = e1 + w1;
        o = make_float2((0.5f * (e0 + e1) - dmin) / rng, (0.5f * (e1 + e2) - dmin) / rng);
    }
    *reinterpret_cast<float2 *>(out + r * 64 + 2 * lane) = o;
}

// AttractorLayerUnnormed (NORMED = false: a_i = softplus(A[., i])) / AttractorLayer (NORMED = true: a_i = relu(A[., 2i]) + 1e-3,
// the A_normed override of attractor.py:104-106) with NA attractors, kind "mean", inverse attractor with alpha 300, gamma 2:
// b_new = b + mean_i dx_i / (1 + 300 dx_i^2), dx_i = a_i - b, b = bilinear_align_corners(b_prev).  Thread layout as
// attractor_kernel: one thread per (pixel, bin), a block = 4 whole pixels.  sort_clip (the last level of the normed head, where
// the centres are consumed): out = clip(sort((max - min) b_new + min), min, max) over the 64 bins of the pixel, sorted by a
// bitonic network in shared memory; otherwise out = b_new (the next level's b_prev, unsorted as in the reference).
template <int NA, bool NORMED>
__global__ void __launch_bounds__(256) attractor_single_kernel(const float *__restrict__ A, int lda, const float *__restrict__ bprev, int Hp, int Wp,
                                                               int H, int W, float sy, float sx, int sort_clip, float dmin, float dmax,
                                                               float *__restrict__ bout) {
    __shared__ float s_c[256];
    const int y = blockIdx.y, f = blockIdx.z;
    const int t = blockIdx.x * 256 + threadIdx.x;
    const int x = t >> 6, k = t & 63;
    const int lane = threadIdx.x & 31;
    const bool ok = x < W;
    const int xc = ok ? x : W - 1;
    const float fy = sy * (float)y, fx = sx * (float)xc;
    const int y0 = min((int)fy, Hp - 1), x0 = min((int)fx, Wp - 1);
    const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const float *bp = bprev + (size_t)f * Hp * Wp * 64 + k;
    const float b = hy * (hx * bp[(size_t)(y0 * Wp + x0) * 64] + lx * bp[(size_t)(y0 * Wp + x1) * 64]) +
                    ly * (hx * bp[(size_t)(y1 * Wp + x0) * 64] + lx * bp[(size_t)(y1 * Wp + x1) * 64]);
    const float *arow = A + ((size_t)(f * H + y) * W + xc) * lda;
    const int ai = lane & (NA - 1);                      // lanes 0..NA-1 hold the pixel's attractor points
    const float a_mine = NORMED ? fmaxf(arow[2 * ai], 0.f) + 1e-3f : softplus_f(arow[ai]);
    float delta = 0.f;
#pragma unroll
    for (int i = 0; i < NA; ++i) {
        const float dx = __shfl_sync(0xffffffffu, a_mine, i) - b;
        delta += __fdividef(dx, 1.f + 300.f * (dx * dx));
    }
    const float bn = b + delta / (float)NA;
    const size_t o = ((size_t)(f * H + y) * W + x) * 64 + k;
    if (!NORMED || !sort_clip) {
        if (ok) bout[o] = bn;
        return;
    }
    s_c[threadIdx.x] = (dmax - dmin) * bn + dmin;        // sort_clip is uniform over the grid: every thread reaches the barriers
    __syncthreads();
    const int base = threadIdx.x & ~63;
#pragma unroll
    for (int size = 2; size <= 64; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const int partner = k ^ stride;
            if (partner > k) {
                const float u = s_c[base + k], v = s_c[base + partner];
                if ((u > v) == ((k & size) == 0)) { s_c[base + k] = v; s_c[base + partner] = u; }
            }
            __syncthreads();
        }
    }
    if (ok) bout[o] = fminf(fmaxf(s_c[threadIdx.x], dmin), dmax);
}

// ConditionalLogBinomial(33, 128, 64) + expectation of the single head, per net pixel: as clb_final_kernel, with 33 main inputs
// (the 32 out_conv channels and the core's relative depth, zoedepth_v1.py:171-186) and an 80-wide hidden layer.  The relative depth
// is the DPT output at the same size, relu(wr . out_conv + br) (base_models/midas.py:268), computed here from the out_conv values
// this thread reads anyway.
constexpr int CLB1_IN = 33, CLB1_HID = 80;
struct ClbSingleParams {
    const __half *o32; int ldo;          // [F, nh, nw, ldo] relu'd out_conv activation, channels 0..31
    const float *ze; int ldz;            // [F, h3, w3, ldz]: W_e . b_emb, columns 0..79
    const float *bc;                     // [F, h3, w3, 64] bin centres
    const float *wo;                     // [33][80] (input channel major; row 32 = relative depth)
    const float *b0;                     // [80]
    const float *w2;                     // [4][80]
    const float *b2;                     // [4]
    const float *wr; float br;           // [32], scalar: the core's final 1x1 conv
    int F, nh, nw, h3, w3;
    float sy, sx, min_temp, max_temp;
    float *out;                          // [F, nh, nw]
};

__global__ void __launch_bounds__(128) clb_single_kernel(ClbSingleParams p) {
    __shared__ float s_wo[CLB1_IN * CLB1_HID], s_b0[CLB1_HID], s_w2[4 * CLB1_HID], s_b2[4], s_lb[64], s_wr[32];
    const int f = blockIdx.z;
    for (int i = threadIdx.x; i < CLB1_IN * CLB1_HID; i += 128) s_wo[i] = p.wo[i];
    for (int i = threadIdx.x; i < 4 * CLB1_HID; i += 128) s_w2[i] = p.w2[i];
    if (threadIdx.x < CLB1_HID) s_b0[threadIdx.x] = p.b0[threadIdx.x];
    if (threadIdx.x < 4) s_b2[threadIdx.x] = p.b2[threadIdx.x];
    if (threadIdx.x < 64) s_lb[threadIdx.x] = log_binom_f(63.f, (float)threadIdx.x);
    if (threadIdx.x < 32) s_wr[threadIdx.x] = p.wr[threadIdx.x];
    __syncthreads();
    const int y = blockIdx.y, x = blockIdx.x * 128 + threadIdx.x;
    if (x >= p.nw) return;
    const float fy = p.sy * (float)y, fx = p.sx * (float)x;
    const int y0 = min((int)fy, p.h3 - 1), y1 = min(y0 + 1, p.h3 - 1), x0 = min((int)fx, p.w3 - 1), x1 = min(x0 + 1, p.w3 - 1);
    const float ly = fy - (float)y0, hy = 1.f - ly, lx = fx - (float)x0, hx = 1.f - lx;
    const size_t i00 = ((size_t)f * p.h3 + y0) * p.w3 + x0, i01 = ((size_t)f * p.h3 + y0) * p.w3 + x1;
    const size_t i10 = ((size_t)f * p.h3 + y1) * p.w3 + x0, i11 = ((size_t)f * p.h3 + y1) * p.w3 + x1;
    float pre[CLB1_HID];
    {
        const float4 *z00 = reinterpret_cast<const float4 *>(p.ze + i00 * p.ldz), *z01 = reinterpret_cast<const float4 *>(p.ze + i01 * p.ldz);
        const float4 *z10 = reinterpret_cast<const float4 *>(p.ze + i10 * p.ldz), *z11 = reinterpret_cast<const float4 *>(p.ze + i11 * p.ldz);
#pragma unroll
        for (int k = 0; k < CLB1_HID / 4; ++k) {
            const float4 a = __ldg(z00 + k), b = __ldg(z01 + k), c = __ldg(z10 + k), d = __ldg(z11 + k);
            pre[4 * k + 0] = s_b0[4 * k + 0] + (hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x));
            pre[4 * k + 1] = s_b0[4 * k + 1] + (hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y));
            pre[4 * k + 2] = s_b0[4 * k + 2] + (hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z));
            pre[4 * k + 3] = s_b0[4 * k + 3] + (hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w));
        }
    }
    float rel = 0.f;
    {
        const uint4 *op = reinterpret_cast<const uint4 *>(p.o32 + (((size_t)f * p.nh + y) * p.nw + x) * p.ldo);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint4 u = __ldg(op + q);
            const __half2 *h2 = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 o2 = __half22float2(h2[e]);
                const int c = q * 8 + 2 * e;
                rel = fmaf(s_wr[c + 1], o2.y, fmaf(s_wr[c], o2.x, rel));
                const float *w0 = s_wo + c * CLB1_HID, *w1 = w0 + CLB1_HID;
#pragma unroll
                for (int k = 0; k < CLB1_HID; ++k) pre[k] = fmaf(w1[k], o2.y, fmaf(w0[k], o2.x, pre[k]));
            }
        }
    }
    rel = fmaxf(rel + p.br, 0.f);
    {
        const float *wrel = s_wo + 32 * CLB1_HID;
#pragma unroll
        for (int k = 0; k < CLB1_HID; ++k) pre[k] = fmaf(wrel[k], rel, pre[k]);
    }
    float pt[4] = {s_b2[0], s_b2[1], s_b2[2], s_b2[3]};
#pragma unroll
    for (int k = 0; k < CLB1_HID; ++k) {
        const float g = 0.5f * pre[k] * (1.f + erff(pre[k] * 0.70710678118654752f));                 // nn.GELU (erf form)
#pragma unroll
        for (int j = 0; j < 4; ++j) pt[j] = fmaf(s_w2[j * CLB1_HID + k], g, pt[j]);
    }
    const float pa = softplus_f(pt[0]) + 1e-4f, pb = softplus_f(pt[1]) + 1e-4f, ta = softplus_f(pt[2]) + 1e-4f, tb = softplus_f(pt[3]) + 1e-4f;
    const float prob = pa / (pa + pb);
    const float temp = (p.max_temp - p.min_temp) * (ta / (ta + tb)) + p.min_temp;
    const float lp = logf(fminf(fmaxf(prob, 1e-4f), 1.f)), lq = logf(fminf(fmaxf(1.f - prob, 1e-4f), 1.f));
    const float inv_t = 1.f / temp;
    float mx = -INFINITY;
#pragma unroll 8
    for (int k = 0; k < 64; ++k) mx = fmaxf(mx, (s_lb[k] + (float)k * lp + (float)(63 - k) * lq) * inv_t);
    const float4 *c00 = reinterpret_cast<const float4 *>(p.bc + i00 * 64), *c01 = reinterpret_cast<const float4 *>(p.bc + i01 * 64);
    const float4 *c10 = reinterpret_cast<const float4 *>(p.bc + i10 * 64), *c11 = reinterpret_cast<const float4 *>(p.bc + i11 * 64);
    float den = 0.f, num = 0.f;
#pragma unroll 4
    for (int k4 = 0; k4 < 16; ++k4) {
        const float4 a = __ldg(c00 + k4), b = __ldg(c01 + k4), c = __ldg(c10 + k4), d = __ldg(c11 + k4);
        const float bcv[4] = {hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x), hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y),
                              hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z), hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w)};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 4 * k4 + e;
            const float ek = expf((s_lb[k] + (float)k * lp + (float)(63 - k) * lq) * inv_t - mx);
            den += ek;
            num = fmaf(ek, bcv[e], num);
        }
    }
    p.out[((size_t)f * p.nh + y) * p.nw + x] = num / den;
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

DM_EXPORT int dm_zoe_preprocess_patchify(const uint8_t *rgb, int B, int H, int W, int pad_h, int pad_w, int net_h, int net_w, int patch,
                                         void *out, int kpad, void *stream_) {
    using namespace dm;
    if (!rgb || !out || net_h % patch || net_w % patch || kpad != 3 * patch * patch || pad_h >= H || pad_w >= W || pad_h < 0 || pad_w < 0) {
        set_error("dm_zoe_preprocess_patchify: bad arguments (reflect padding must be smaller than the image; kpad = 3*patch^2)");
        return DM_E_INVALID;
    }
    ZoePre p;
    p.rgb = rgb; p.B = B; p.H = H; p.W = W; p.pad_h = pad_h; p.pad_w = pad_w; p.nh = net_h; p.nw = net_w; p.patch = patch;
    p.gh = net_h / patch; p.gw = net_w / patch; p.kpad = kpad; p.out = (__half *)out;
    const long long total = (long long)2 * B * net_h * net_w;
    zoe_preprocess_patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("zoe_preprocess_patchify_kernel");
    return DM_OK;
}

DM_EXPORT int dm_layernorm_post_f16(float *x, long long rows, int C, const float *gamma, const float *beta, float eps, void *out, void *stream_) {
    using namespace dm;
    if (C != 128) { set_error("dm_layernorm_post_f16: width must be 128 (router embedding)"); return DM_E_UNSUPPORTED; }
    layernorm_post_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream_>>>(x, rows, gamma, beta, eps, (__half *)out);
    DM_LAUNCH_CHECK("layernorm_post_kernel");
    return DM_OK;
}

DM_EXPORT int dm_attention_small_f16(const void *qkv, int F, int S, int heads, float scale, void *out, void *stream_) {
    using namespace dm;
    const size_t smem = ((size_t)2 * S * RA_PITCH + (size_t)8 * S) * sizeof(float);
    if (smem > 200 * 1024) { set_error("dm_attention_small_f16: %d tokens do not fit in shared memory", S); return DM_E_UNSUPPORTED; }
    if (smem > 48 * 1024) {
        static PerDeviceFlag configured;
        if (!configured.test_and_set())
            DM_CUDA_CHECK(cudaFuncSetAttribute(attention_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    attention_small_kernel<<<dim3(F, heads, 4), 256, smem, (cudaStream_t)stream_>>>((const __half *)qkv, S, heads * RA_HD, scale, (__half *)out);   // 4 query-row blocks per (forward, head)
    DM_LAUNCH_CHECK("attention_small_kernel");
    return DM_OK;
}

DM_EXPORT int dm_cast_f32_f16(const float *x, long long n, void *out, void *stream_) {
    using namespace dm;
    if (n % 4) { set_error("dm_cast_f32_f16: element count must be a multiple of 4"); return DM_E_INVALID; }
    cast_f32_f16_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(x, n / 4, (__half *)out);
    DM_LAUNCH_CHECK("cast_f32_f16_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_select_softplus(const float *seed, int ld, const float *logits, int lld, int F, int rows_per_fwd, float *out, void *stream_) {
    using namespace dm;
    const long long rows = (long long)F * rows_per_fwd;
    select_softplus_kernel<<<(unsigned)((rows * 64 + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(seed, ld, logits, lld, rows, rows_per_fwd, out);
    DM_LAUNCH_CHECK("select_softplus_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_add_nhwc_f16(const void *a, const void *b_small, int B, int Hs, int Ws, int C, void *out, int H, int W, void *stream_) {
    using namespace dm;
    if (C % 8 || H > 65535 || B > 65535) { set_error("dm_resize_add_nhwc_f16: bad shape"); return DM_E_INVALID; }
    const float sy = H > 1 ? (float)(Hs - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Ws - 1) / (float)(W - 1) : 0.f;
    const dim3 grid((unsigned)((W * (C / 8) + 255) / 256), (unsigned)H, (unsigned)B);
    resize_add_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __half *)a, (const __half *)b_small, Hs, Ws, C, (__half *)out, H, W, sy, sx);
    DM_LAUNCH_CHECK("resize_add_nhwc_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_attractor(const float *A, int lda, const float *logits, int lld, const float *b_prev, int F, int Hp, int Wp, int H, int W,
                               float *b_out, void *stream_) {
    using namespace dm;
    if (H > 65535 || F > 65535) { set_error("dm_zoe_attractor: bad shape"); return DM_E_INVALID; }
    const float sy = H > 1 ? (float)(Hp - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Wp - 1) / (float)(W - 1) : 0.f;
    const dim3 grid((unsigned)((W * 64 + 255) / 256), (unsigned)H, (unsigned)F);
    attractor_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>(A, lda, logits, lld, b_prev, Hp, Wp, H, W, sy, sx, b_out);
    DM_LAUNCH_CHECK("attractor_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_clb_final(const void *o32, int ldo, const float *ze, int ldz, const float *bc, const float *logits, int lld, const float *wo,
                               const float *b0, const float *w2, const float *b2, int F, int nh, int nw, int h3, int w3, float min_temp,
                               float max_temp, float *out, void *stream_) {
    using namespace dm;
    if (nh > 65535 || F > 65535) { set_error("dm_zoe_clb_final: bad shape"); return DM_E_INVALID; }
    ClbParams p;
    p.o32 = (const __half *)o32; p.ldo = ldo; p.ze = ze; p.ldz = ldz; p.bc = bc; p.logits = logits; p.lld = lld;
    p.wo = wo; p.b0 = b0; p.w2 = w2; p.b2 = b2; p.F = F; p.nh = nh; p.nw = nw; p.h3 = h3; p.w3 = w3;
    p.sy = nh > 1 ? (float)(h3 - 1) / (float)(nh - 1) : 0.f;
    p.sx = nw > 1 ? (float)(w3 - 1) / (float)(nw - 1) : 0.f;
    p.min_temp = min_temp; p.max_temp = max_temp; p.out = out;
    if (ldo % 8 || ldz % 4) { set_error("dm_zoe_clb_final: ldo must be a multiple of 8 and ldz of 4"); return DM_E_INVALID; }
    clb_final_kernel<<<dim3((unsigned)((nw + 127) / 128), (unsigned)nh, (unsigned)F), 128, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("clb_final_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_tta_combine(const float *d, int B, int nh, int nw, int pad_h, int pad_w, int H, int W, float *out, void *stream_) {
    using namespace dm;
    const long long total = (long long)B * H * W;
    tta_combine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(d, B, nh, nw, H + 2 * pad_h, W + 2 * pad_w, pad_h, pad_w, H, W, out);
    DM_LAUNCH_CHECK("tta_combine_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_seed_bins(const float *seed, int ld, long long rows, int normed, float min_depth, float max_depth, float *out, void *stream_) {
    using namespace dm;
    if (!seed || !out || rows < 0 || ld < 64 || ld % 2 || (normed != 0 && normed != 1) || (normed && !(max_depth > min_depth))) {
        set_error("dm_zoe_seed_bins: bad arguments (ld >= 64 and even, normed 0 / 1, max_depth > min_depth)");
        return DM_E_INVALID;
    }
    if (rows == 0) return DM_OK;
    seed_bins_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream_>>>(seed, ld, rows, normed, min_depth, max_depth, out);
    DM_LAUNCH_CHECK("seed_bins_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_attractor_single(const float *A, int lda, int n_attractors, int normed, const float *b_prev, int F, int Hp, int Wp, int H,
                                      int W, int sort_clip, float min_depth, float max_depth, float *b_out, void *stream_) {
    using namespace dm;
    if (n_attractors != 16 && n_attractors != 8 && n_attractors != 4 && n_attractors != 1) {
        set_error("dm_zoe_attractor_single: %d attractors (implemented: 16, 8, 4, 1)", n_attractors);
        return DM_E_UNSUPPORTED;
    }
    if (!A || !b_prev || !b_out || (normed != 0 && normed != 1) || (sort_clip != 0 && sort_clip != 1) || (sort_clip && !normed) ||
        lda < (normed ? 2 : 1) * n_attractors || F < 1 || Hp < 1 || Wp < 1 || H < 1 || W < 1 || H > 65535 || F > 65535 ||
        (normed && !(max_depth > min_depth))) {
        set_error("dm_zoe_attractor_single: bad arguments (lda >= %d, sort_clip only for the normed head, max_depth > min_depth)",
                  (normed ? 2 : 1) * n_attractors);
        return DM_E_INVALID;
    }
    const float sy = H > 1 ? (float)(Hp - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Wp - 1) / (float)(W - 1) : 0.f;
    const dim3 grid((unsigned)((W * 64 + 255) / 256), (unsigned)H, (unsigned)F);
    cudaStream_t st = (cudaStream_t)stream_;
#define DM_ATT1(NA, NORMED) attractor_single_kernel<NA, NORMED><<<grid, 256, 0, st>>>(A, lda, b_prev, Hp, Wp, H, W, sy, sx, sort_clip, min_depth, max_depth, b_out)
    switch (n_attractors * 2 + normed) {
        case 32: DM_ATT1(16, false); break;
        case 33: DM_ATT1(16, true); break;
        case 16: DM_ATT1(8, false); break;
        case 17: DM_ATT1(8, true); break;
        case 8: DM_ATT1(4, false); break;
        case 9: DM_ATT1(4, true); break;
        case 2: DM_ATT1(1, false); break;
        default: DM_ATT1(1, true); break;
    }
#undef DM_ATT1
    DM_LAUNCH_CHECK("attractor_single_kernel");
    return DM_OK;
}

DM_EXPORT int dm_zoe_clb_single(const void *o32, int ldo, const float *ze, int ldz, const float *bc, const float *wo, const float *b0, const float *w2,
                                const float *b2, const float *wr, float br, int F, int nh, int nw, int h3, int w3, float min_temp, float max_temp,
                                float *out, void *stream_) {
    using namespace dm;
    if (!o32 || !ze || !bc || !wo || !b0 || !w2 || !b2 || !wr || !out || F < 1 || nh < 1 || nw < 1 || h3 < 1 || w3 < 1 || nh > 65535 || F > 65535) {
        set_error("dm_zoe_clb_single: bad shape or null pointer");
        return DM_E_INVALID;
    }
    if (ldo % 8 || ldo < 32 || ldz % 4 || ldz < CLB1_HID) {
        set_error("dm_zoe_clb_single: ldo must be a multiple of 8 and >= 32, ldz a multiple of 4 and >= %d", CLB1_HID);
        return DM_E_INVALID;
    }
    ClbSingleParams p;
    p.o32 = (const __half *)o32; p.ldo = ldo; p.ze = ze; p.ldz = ldz; p.bc = bc;
    p.wo = wo; p.b0 = b0; p.w2 = w2; p.b2 = b2; p.wr = wr; p.br = br; p.F = F; p.nh = nh; p.nw = nw; p.h3 = h3; p.w3 = w3;
    p.sy = nh > 1 ? (float)(h3 - 1) / (float)(nh - 1) : 0.f;
    p.sx = nw > 1 ? (float)(w3 - 1) / (float)(nw - 1) : 0.f;
    p.min_temp = min_temp; p.max_temp = max_temp; p.out = out;
    clb_single_kernel<<<dim3((unsigned)((nw + 127) / 128), (unsigned)nh, (unsigned)F), 128, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("clb_single_kernel");
    return DM_OK;
}
