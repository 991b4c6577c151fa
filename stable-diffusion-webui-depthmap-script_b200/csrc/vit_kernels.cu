// Bandwidth-bound kernels around the tensor-core GEMMs of the depth networks (all coalesced / vectorised, fp32 math):
//   preprocess_patchify  uint8 image -> [cv2-style bicubic resize] -> normalise -> fp16 patch matrix (im2col of the
//                        patch-embedding conv; reference: depth_anything_v2/dpt.py:196-221 + util/transform.py,
//                        dmidas/transforms.py:48-231, dinov2_layers/patch_embed.py:76, dmidas/backbones/beit.py:18-26)
//   preprocess_patchify_f32_crops  the same for B crops of one planar fp32 image (BOOST's estimatemidasBoost,
//                        src/depthmap_generation.py:1180-1203: cubic resize of the float crop, ImageNet mean / std)
//   assemble_tokens      [cls | patch tokens] + positional embedding -> fp32 residual stream (dinov2.py:212-216)
//   layernorm_f16        fp32 residual stream -> LayerNorm -> fp16 GEMM operand (eps 1e-6), optional "drop cls" remap
//   resize_bilinear_nhwc fp16 NHWC bilinear, align_corners=True (util/blocks.py:143, dmidas/blocks.py:433)
//   resize_f32           final depth resize: bilinear align_corners=True (DA-v2, src/depthmap_generation.py:558) or
//                        bicubic align_corners=False (MiDaS, :487-497)
//   im2col_s2            3x3 stride-2 pad-1 gather for the one strided conv of the reassemble stage (dpt.py:75-80)
// Split variants (the fp32-class path of no_half, gemm_wgmma.cu): the patch matrix, LayerNorm output and NHWC resize store an
// fp32 value v as fp16 hi = rn(v), lo = rn(v - hi) in rows [hi | lo | hi] of 3x the width; the assembly reads an fp32 patch
// embedding.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "cv_cubic.cuh"

namespace dm {

// ---------------------------------------------------------------------------------------------------------------
// preprocess + patchify
// ---------------------------------------------------------------------------------------------------------------
struct PreParams {
    const uint8_t *rgb;  // [B, H, W, 3]
    int B, H, W;         // source image
    int nh, nw;          // network input size (multiple of patch)
    int patch, gh, gw;   // patch size, grid
    int kpad;            // padded K (>= 3*patch*patch, multiple of 64)
    float mean[3], inv_std[3];
    int chan_map[3];     // network channel c reads source channel chan_map[c]
    __half *out;         // [B*gh*gw, kpad]; split: [B*gh*gw, 3*kpad], rows [hi | lo | hi]
};

// normalise network pixel (y, x) of image b and store it into its patch row, K ordered (c, ky, kx)
template <bool SPLIT = false>
__device__ __forceinline__ void store_patch_pixel(const PreParams &p, int b, int y, int x, const float (&v)[3], float value_scale) {
    const int py = y / p.patch, ky = y % p.patch, pxi = x / p.patch, kx = x % p.patch;
    __half *row = p.out + ((long long)(b * p.gh + py) * p.gw + pxi) * (SPLIT ? 3 * p.kpad : p.kpad);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float val = (v[p.chan_map[c]] * value_scale - p.mean[c]) * p.inv_std[c];
        const int k = (c * p.patch + ky) * p.patch + kx;
        const __half hi = __float2half_rn(val);
        row[k] = hi;
        if (SPLIT) {
            row[p.kpad + k] = __float2half_rn(val - __half2float(hi));
            row[2 * p.kpad + k] = hi;
        }
    }
}

template <bool SPLIT>
__global__ void __launch_bounds__(256) preprocess_patchify_kernel(PreParams p) {
    // one thread per (network pixel, channel triple): thread -> (b, y, x) of the network input
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)p.B * p.nh * p.nw;
    if (idx >= total) return;
    const int x = (int)(idx % p.nw);
    const int y = (int)((idx / p.nw) % p.nh);
    const int b = (int)(idx / ((long long)p.nw * p.nh));
    const U8Source src{p.rgb + (long long)b * p.H * p.W * 3, p.H, p.W};
    float v[3];
    cubic_sample(src, p.nh, p.nw, y, x, v);
    store_patch_pixel<SPLIT>(p, b, y, x, v, 1.0f / 255.0f);
}

// ragged batch: image b is desc[b] of the packed buffer p.rgb (p.H, p.W unused)
template <bool SPLIT>
__global__ void __launch_bounds__(256) preprocess_patchify_ragged_kernel(PreParams p, const dm_ragged_image *__restrict__ desc) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)p.B * p.nh * p.nw;
    if (idx >= total) return;
    const int x = (int)(idx % p.nw);
    const int y = (int)((idx / p.nw) % p.nh);
    const int b = (int)(idx / ((long long)p.nw * p.nh));
    const dm_ragged_image d = desc[b];
    const U8Source src{p.rgb + d.offset, d.h, d.w};
    float v[3];
    cubic_sample(src, p.nh, p.nw, y, x, v);
    store_patch_pixel<SPLIT>(p, b, y, x, v, 1.0f / 255.0f);
}

// BOOST crops: p.rgb unused; image b is the crop rects[b] = (x0, y0, w, h) of the planar fp32 image, values used as they are
__global__ void __launch_bounds__(256) preprocess_patchify_f32_crops_kernel(PreParams p, const float *__restrict__ img, int Hi, int Wi,
                                                                            const int *__restrict__ rects) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)p.B * p.nh * p.nw;
    if (idx >= total) return;
    const int x = (int)(idx % p.nw);
    const int y = (int)((idx / p.nw) % p.nh);
    const int b = (int)(idx / ((long long)p.nw * p.nh));
    const int4 r = __ldg(reinterpret_cast<const int4 *>(rects) + b);
    const F32CropSource src{img + (long long)r.y * Wi + r.x, (long long)Hi * Wi, Wi, r.w, r.z};
    float v[3];
    cubic_sample(src, p.nh, p.nw, y, x, v);
    store_patch_pixel(p, b, y, x, v, 1.0f);
}

__global__ void zero_pad_cols_kernel(__half *out, long long rows, int kused, int kpad) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int padw = kpad - kused;
    if (idx >= rows * padw) return;
    out[(idx / padw) * kpad + kused + (idx % padw)] = __float2half_rn(0.f);
}

// ---------------------------------------------------------------------------------------------------------------
// tokens = [cls ; patch embeddings] + pos
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) assemble_tokens_kernel(const T *__restrict__ pe, const float *__restrict__ cls,
                                                              const float *__restrict__ pos, float *__restrict__ X, int B, int Np, int C) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per 4 channels
    const int c4 = C / 4;
    const long long total = (long long)B * (Np + 1) * c4;
    if (idx >= total) return;
    const int c = (int)(idx % c4) * 4;
    const long long row = idx / c4;
    const int t = (int)(row % (Np + 1));
    const int b = (int)(row / (Np + 1));
    float4 v;
    if (t == 0) v = *reinterpret_cast<const float4 *>(cls + c);
    else if constexpr (sizeof(T) == 4) {
        v = *reinterpret_cast<const float4 *>(pe + ((long long)b * Np + (t - 1)) * C + c);
    } else {
        const __half2 *h = reinterpret_cast<const __half2 *>(pe + ((long long)b * Np + (t - 1)) * C + c);
        const float2 a = __half22float2(h[0]), d = __half22float2(h[1]);
        v = make_float4(a.x, a.y, d.x, d.y);
    }
    if (pos) {
        const float4 q = *reinterpret_cast<const float4 *>(pos + (long long)t * C + c);
        v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    }
    *reinterpret_cast<float4 *>(X + row * C + c) = v;
}

// four consecutive fp32 values as split fp16: hi at dst, lo at dst + lo_off, hi again at dst + 2 lo_off (8-byte stores)
__device__ __forceinline__ void store_split4(__half *dst, long long lo_off, const float (&y)[4]) {
    const __half2 h0 = __floats2half2_rn(y[0], y[1]), h1 = __floats2half2_rn(y[2], y[3]);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    const __half2 l0 = __floats2half2_rn(y[0] - f0.x, y[1] - f0.y), l1 = __floats2half2_rn(y[2] - f1.x, y[3] - f1.y);
    uint2 hu, lu;
    hu.x = *reinterpret_cast<const uint32_t *>(&h0); hu.y = *reinterpret_cast<const uint32_t *>(&h1);
    lu.x = *reinterpret_cast<const uint32_t *>(&l0); lu.y = *reinterpret_cast<const uint32_t *>(&l1);
    *reinterpret_cast<uint2 *>(dst) = hu;
    *reinterpret_cast<uint2 *>(dst + lo_off) = lu;
    *reinterpret_cast<uint2 *>(dst + 2 * lo_off) = hu;
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, fp32 two-pass statistics in registers, fp16 output
// ---------------------------------------------------------------------------------------------------------------
template <int VEC, bool SPLIT = false>  // float4 loads per lane: C = 128 * VEC; SPLIT: rows of 3C, [hi | lo | hi]
__global__ void __launch_bounds__(256) layernorm_f16_kernel(const float *__restrict__ x, long long rows, int C, const float *__restrict__ gamma,
                                                            const float *__restrict__ beta, float eps, __half *__restrict__ out,
                                                            int tokens_per_img, int drop_first) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows) return;
    long long orow = row;
    if (drop_first) {
        const long long b = row / tokens_per_img;
        const int t = (int)(row % tokens_per_img);
        if (t == 0) return;
        orow = b * (tokens_per_img - 1) + (t - 1);
    }
    const float4 *xr = reinterpret_cast<const float4 *>(x + row * C);
    float4 v[VEC];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) { v[i] = xr[lane + 32 * i]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const float a = v[i].x - mean, b2 = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b2 * b2) + (c * c + d * d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)C + eps);
    __half *orow_p = out + orow * (SPLIT ? 3 * C : C);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c = (lane + 32 * i) * 4;
        const float4 g = *reinterpret_cast<const float4 *>(gamma + c), bt = *reinterpret_cast<const float4 *>(beta + c);
        if (SPLIT) {
            const float y[4] = {(v[i].x - mean) * rstd * g.x + bt.x, (v[i].y - mean) * rstd * g.y + bt.y,
                                (v[i].z - mean) * rstd * g.z + bt.z, (v[i].w - mean) * rstd * g.w + bt.w};
            store_split4(orow_p + c, C, y);
            continue;
        }
        const __half2 h0 = __floats2half2_rn((v[i].x - mean) * rstd * g.x + bt.x, (v[i].y - mean) * rstd * g.y + bt.y);
        const __half2 h1 = __floats2half2_rn((v[i].z - mean) * rstd * g.z + bt.z, (v[i].w - mean) * rstd * g.w + bt.w);
        uint2 u;
        u.x = *reinterpret_cast<const uint32_t *>(&h0);
        u.y = *reinterpret_cast<const uint32_t *>(&h1);
        *reinterpret_cast<uint2 *>(orow_p + c) = u;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// bilinear resize, NHWC fp16, align_corners=True; one thread per (output pixel, 8 channels)
// ---------------------------------------------------------------------------------------------------------------
// grid = (ceil(Wout * C/8 / 256), Hout, B): the row and image come from the block index, so the only division left is the
// 32-bit x = t / (C/8) (the first version spent most of its time in 64-bit div/mod of a flat index and ran at a quarter
// of the HBM rate).  One thread = 8 channels of one output pixel: four 16-byte loads (L1/L2 hits: every input pixel is
// read by ~4 x scale^2 threads), one 16-byte store.
__global__ void __launch_bounds__(256) resize_bilinear_nhwc_kernel(const __half *__restrict__ in, int Hin, int Win, int C,
                                                                   __half *__restrict__ out, int Hout, int Wout, float sy, float sx) {
    const int c8 = C >> 3;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= Wout * c8) return;
    const int x = t / c8;
    const int c = (t - x * c8) << 3;
    const int y = blockIdx.y, b = blockIdx.z;
    const float fy = sy * (float)y, fx = sx * (float)x;
    const int y0 = min((int)fy, Hin - 1), x0 = min((int)fx, Win - 1);
    const int y1 = min(y0 + 1, Hin - 1), x1 = min(x0 + 1, Win - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const __half *base = in + (size_t)b * Hin * Win * C + c;
    const uint4 u00 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y0 * Win + x0) * C));
    const uint4 u01 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y0 * Win + x1) * C));
    const uint4 u10 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y1 * Win + x0) * C));
    const uint4 u11 = __ldg(reinterpret_cast<const uint4 *>(base + (size_t)(y1 * Win + x1) * C));
    const __half2 *a = reinterpret_cast<const __half2 *>(&u00), *bq = reinterpret_cast<const __half2 *>(&u01);
    const __half2 *cq = reinterpret_cast<const __half2 *>(&u10), *d = reinterpret_cast<const __half2 *>(&u11);
    uint4 o;
    __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 f00 = __half22float2(a[k]), f01 = __half22float2(bq[k]), f10 = __half22float2(cq[k]), f11 = __half22float2(d[k]);
        // torch upsample_bilinear2d: hy*(hx*v00 + lx*v01) + ly*(hx*v10 + lx*v11)
        const float r0 = hy * (hx * f00.x + lx * f01.x) + ly * (hx * f10.x + lx * f11.x);
        const float r1 = hy * (hx * f00.y + lx * f01.y) + ly * (hx * f10.y + lx * f11.y);
        oh[k] = __floats2half2_rn(r0, r1);
    }
    __stcs(reinterpret_cast<uint4 *>(out + ((size_t)(b * Hout + y) * Wout + x) * C + c), o);
}

// the same on split tensors [B, H, W, 3C]: one thread per (output pixel, 4 channels), hi + lo interpolated in fp32, re-split
__global__ void __launch_bounds__(256) resize_bilinear_nhwc_split_kernel(const __half *__restrict__ in, int Hin, int Win, int C,
                                                                         __half *__restrict__ out, int Hout, int Wout, float sy, float sx) {
    const int c4 = C >> 2;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= Wout * c4) return;
    const int x = t / c4;
    const int c = (t - x * c4) << 2;
    const int y = blockIdx.y, b = blockIdx.z;
    const float fy = sy * (float)y, fx = sx * (float)x;
    const int y0 = min((int)fy, Hin - 1), x0 = min((int)fx, Win - 1);
    const int y1 = min(y0 + 1, Hin - 1), x1 = min(x0 + 1, Win - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const __half *base = in + (size_t)b * Hin * Win * 3 * C + c;
    const size_t px[4] = {(size_t)(y0 * Win + x0) * 3 * C, (size_t)(y0 * Win + x1) * 3 * C, (size_t)(y1 * Win + x0) * 3 * C,
                          (size_t)(y1 * Win + x1) * 3 * C};
    float f[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint2 hu = __ldg(reinterpret_cast<const uint2 *>(base + px[q])), lu = __ldg(reinterpret_cast<const uint2 *>(base + px[q] + C));
        const float2 h0 = __half22float2(*reinterpret_cast<const __half2 *>(&hu.x)), h1 = __half22float2(*reinterpret_cast<const __half2 *>(&hu.y));
        const float2 l0 = __half22float2(*reinterpret_cast<const __half2 *>(&lu.x)), l1 = __half22float2(*reinterpret_cast<const __half2 *>(&lu.y));
        f[q][0] = h0.x + l0.x; f[q][1] = h0.y + l0.y; f[q][2] = h1.x + l1.x; f[q][3] = h1.y + l1.y;
    }
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = hy * (hx * f[0][k] + lx * f[1][k]) + ly * (hx * f[2][k] + lx * f[3][k]);
    store_split4(out + ((size_t)(b * Hout + y) * Wout + x) * 3 * C + c, C, r);
}

// single-channel fp32 resize: mode 0 = bilinear align_corners=True, mode 1 = bicubic align_corners=False (A = -0.75)
// `ld` = distance between consecutive input pixels in floats (1 for a dense map; N for channel 0 of an [pixels, N] GEMM output)
__global__ void __launch_bounds__(256) resize_f32_kernel(const float *__restrict__ in, int B, int Hin, int Win, float *__restrict__ out,
                                                         int Hout, int Wout, int mode, int ld) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Hout * Wout;
    if (idx >= total) return;
    const int x = (int)(idx % Wout);
    const int y = (int)((idx / Wout) % Hout);
    const int b = (int)(idx / ((long long)Wout * Hout));
    const float *img = in + (long long)b * Hin * Win * ld;
    if (mode == 0) {
        const float sy = Hout > 1 ? (float)(Hin - 1) / (float)(Hout - 1) : 0.f;
        const float sx = Wout > 1 ? (float)(Win - 1) / (float)(Wout - 1) : 0.f;
        const float fy = sy * (float)y, fx = sx * (float)x;
        const int y0 = min((int)fy, Hin - 1), x0 = min((int)fx, Win - 1);
        const int y1 = min(y0 + 1, Hin - 1), x1 = min(x0 + 1, Win - 1);
        const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
        out[idx] = hy * (hx * img[((long long)y0 * Win + x0) * ld] + lx * img[((long long)y0 * Win + x1) * ld]) +
                   ly * (hx * img[((long long)y1 * Win + x0) * ld] + lx * img[((long long)y1 * Win + x1) * ld]);
    } else {
        const float sy = (float)Hin / (float)Hout, sx = (float)Win / (float)Wout;
        float fy = sy * ((float)y + 0.5f) - 0.5f, fx = sx * ((float)x + 0.5f) - 0.5f;
        const int iy = (int)floorf(fy), ix = (int)floorf(fx);
        fy -= (float)iy; fx -= (float)ix;
        float cx[4], cy[4];
        cubic_coeffs(fx, cx);
        cubic_coeffs(fy, cy);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yy = min(max(iy - 1 + j, 0), Hin - 1);
            float r = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) r += cx[i] * img[((long long)yy * Win + min(max(ix - 1 + i, 0), Win - 1)) * ld];
            acc += cy[j] * r;
        }
        out[idx] = acc;
    }
}

// resize_f32_kernel (ld = 1) to a ragged output: image b at its own desc[b] size and place; grid (max h * max w, B)
__global__ void __launch_bounds__(256) resize_f32_ragged_kernel(const float *__restrict__ in, int Hin, int Win, float *__restrict__ out,
                                                                const dm_ragged_image *__restrict__ desc, int mode) {
    const int b = blockIdx.y;
    const dm_ragged_image d = desc[b];
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)d.h * d.w) return;
    const int x = (int)(idx % d.w), y = (int)(idx / d.w);
    const int Hout = d.h, Wout = d.w;
    const float *img = in + (long long)b * Hin * Win;
    float r;
    if (mode == 0) {
        const float sy = Hout > 1 ? (float)(Hin - 1) / (float)(Hout - 1) : 0.f;
        const float sx = Wout > 1 ? (float)(Win - 1) / (float)(Wout - 1) : 0.f;
        const float fy = sy * (float)y, fx = sx * (float)x;
        const int y0 = min((int)fy, Hin - 1), x0 = min((int)fx, Win - 1);
        const int y1 = min(y0 + 1, Hin - 1), x1 = min(x0 + 1, Win - 1);
        const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
        r = hy * (hx * img[(long long)y0 * Win + x0] + lx * img[(long long)y0 * Win + x1]) +
            ly * (hx * img[(long long)y1 * Win + x0] + lx * img[(long long)y1 * Win + x1]);
    } else {
        const float sy = (float)Hin / (float)Hout, sx = (float)Win / (float)Wout;
        float fy = sy * ((float)y + 0.5f) - 0.5f, fx = sx * ((float)x + 0.5f) - 0.5f;
        const int iy = (int)floorf(fy), ix = (int)floorf(fx);
        fy -= (float)iy; fx -= (float)ix;
        float cx[4], cy[4];
        cubic_coeffs(fx, cx);
        cubic_coeffs(fy, cy);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yy = min(max(iy - 1 + j, 0), Hin - 1);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) s += cx[i] * img[(long long)yy * Win + min(max(ix - 1 + i, 0), Win - 1)];
            acc += cy[j] * s;
        }
        r = acc;
    }
    out[d.offset + idx] = r;
}

// im2col for a 3x3 stride-2 pad-1 convolution on NHWC fp16: out [B*Ho*Wo, 9*C] ordered (ky, kx, c).  CIRCULAR: the padding
// wraps around (nn.Conv2d(padding_mode='circular')) instead of being zeros
template <bool CIRCULAR>
__global__ void __launch_bounds__(256) im2col_s2_kernel(const __half *__restrict__ in, int B, int H, int W, int C, __half *__restrict__ out, int Ho, int Wo) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int c8 = C / 8;
    const long long total = (long long)B * Ho * Wo * 9 * c8;
    if (idx >= total) return;
    const int c = (int)(idx % c8) * 8;
    long long r = idx / c8;
    const int tap = (int)(r % 9);
    r /= 9;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho);
    const int b = (int)(r / Ho);
    int y = yo * 2 - 1 + tap / 3, x = xo * 2 - 1 + tap % 3;
    if (CIRCULAR) { y = wrap_index(y, H); x = wrap_index(x, W); }
    uint4 v = make_uint4(0, 0, 0, 0);
    if (y >= 0 && y < H && x >= 0 && x < W) v = __ldg(reinterpret_cast<const uint4 *>(in + (((long long)b * H + y) * W + x) * C + c));
    *reinterpret_cast<uint4 *>(out + ((((long long)b * Ho + yo) * Wo + xo) * 9 + tap) * C + c) = v;
}

// MiDaS ProjectReadout input (dmidas/backbones/utils.py:28-39): row (b, p) = [x[b, 1+p, :], x[b, 0, :]] as fp16
__global__ void __launch_bounds__(256) concat_readout_kernel(const float *__restrict__ x, int B, int N, int C, __half *__restrict__ out) {
    // one block per output row (b, patch p): [ token (b, 1 + p) | class token (b, 0) ] as fp16; 4 channels per thread
    const unsigned row = blockIdx.x;
    const unsigned b = row / (unsigned)(N - 1), p = row - b * (unsigned)(N - 1);
    const float *tok = x + ((size_t)b * N + 1 + p) * C, *cls = x + (size_t)b * N * C;
    __half *dst = out + (size_t)row * (2 * C);
    for (int c = threadIdx.x * 4; c < 2 * C; c += 1024) {
        const float4 v = *reinterpret_cast<const float4 *>(c < C ? tok + c : cls + (c - C));
        const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
        uint2 u;
        u.x = *reinterpret_cast<const uint32_t *>(&h0);
        u.y = *reinterpret_cast<const uint32_t *>(&h1);
        *reinterpret_cast<uint2 *>(dst + c) = u;
    }
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

static int patchify_setup(dm::PreParams &p, int B, int net_h, int net_w, int patch, const float *mean_host, const float *std_host,
                          const int *chan_map_host, void *out, int kpad, cudaStream_t stream) {
    using namespace dm;
    p.B = B; p.nh = net_h; p.nw = net_w; p.patch = patch; p.gh = net_h / patch; p.gw = net_w / patch;
    p.kpad = kpad; p.out = (__half *)out;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; p.chan_map[c] = chan_map_host[c]; }
    const long long rows = (long long)B * p.gh * p.gw;
    const int kused = 3 * patch * patch;
    if (kpad > kused) {
        const long long n = rows * (kpad - kused);
        zero_pad_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((__half *)out, rows, kused, kpad);
        DM_LAUNCH_CHECK("zero_pad_cols_kernel");
    }
    return DM_OK;
}

DM_EXPORT int dm_preprocess_patchify(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, int patch, const float *mean_host,
                                     const float *std_host, const int *chan_map_host, void *out, int kpad, void *stream_) {
    using namespace dm;
    if (!rgb || !out || net_h % patch || net_w % patch || kpad < 3 * patch * patch) { set_error("dm_preprocess_patchify: bad arguments"); return DM_E_INVALID; }
    cudaStream_t stream = (cudaStream_t)stream_;
    PreParams p;
    p.rgb = rgb; p.H = H; p.W = W;
    const int rc = patchify_setup(p, B, net_h, net_w, patch, mean_host, std_host, chan_map_host, out, kpad, stream);
    if (rc) return rc;
    const long long total = (long long)B * net_h * net_w;
    preprocess_patchify_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p);
    DM_LAUNCH_CHECK("preprocess_patchify_kernel");
    return DM_OK;
}

// split patch matrix [B*gh*gw, 3*kpad]: the zero fill treats each row as three rows of kpad
DM_EXPORT int dm_preprocess_patchify_split(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, int patch, const float *mean_host,
                                           const float *std_host, const int *chan_map_host, void *out, int kpad, void *stream_) {
    using namespace dm;
    if (!rgb || !out || net_h % patch || net_w % patch || kpad < 3 * patch * patch) { set_error("dm_preprocess_patchify_split: bad arguments"); return DM_E_INVALID; }
    cudaStream_t stream = (cudaStream_t)stream_;
    PreParams p;
    p.rgb = rgb; p.H = H; p.W = W;
    const int rc = patchify_setup(p, 3 * B, net_h, net_w, patch, mean_host, std_host, chan_map_host, out, kpad, stream);
    if (rc) return rc;
    p.B = B;
    const long long total = (long long)B * net_h * net_w;
    preprocess_patchify_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p);
    DM_LAUNCH_CHECK("preprocess_patchify_kernel");
    return DM_OK;
}

DM_EXPORT int dm_preprocess_patchify_ragged(const uint8_t *packed, long long size, const dm_ragged_image *desc_host, const dm_ragged_image *desc_dev,
                                            int B, int net_h, int net_w, int patch, const float *mean_host, const float *std_host,
                                            const int *chan_map_host, int split, void *out, int kpad, void *stream_) {
    using namespace dm;
    const char *who = "dm_preprocess_patchify_ragged";
    int rc = check_ragged(who, packed, size, desc_host, desc_dev, B, 3, nullptr, nullptr);
    if (rc) return rc;
    if (!out || patch <= 0 || net_h <= 0 || net_w <= 0 || net_h % patch || net_w % patch || kpad < 3 * patch * patch || (split != 0 && split != 1)) {
        set_error("%s: bad arguments", who); return DM_E_INVALID;
    }
    cudaStream_t stream = (cudaStream_t)stream_;
    PreParams p;
    p.rgb = packed; p.H = 0; p.W = 0;
    // split: the zero fill treats each row of 3*kpad as three rows of kpad, as dm_preprocess_patchify_split
    rc = patchify_setup(p, split ? 3 * B : B, net_h, net_w, patch, mean_host, std_host, chan_map_host, out, kpad, stream);
    if (rc) return rc;
    p.B = B;
    const long long total = (long long)B * net_h * net_w;
    if (split) preprocess_patchify_ragged_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p, desc_dev);
    else preprocess_patchify_ragged_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p, desc_dev);
    DM_LAUNCH_CHECK("preprocess_patchify_ragged_kernel");
    return DM_OK;
}

DM_EXPORT int dm_preprocess_patchify_f32_crops(const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w, int patch,
                                               const float *mean_host, const float *std_host, const int *chan_map_host, void *out, int kpad,
                                               void *stream_) {
    using namespace dm;
    if (!img || !rects_dev || !out || B <= 0 || Hi <= 0 || Wi <= 0 || net_h % patch || net_w % patch || kpad < 3 * patch * patch) {
        set_error("dm_preprocess_patchify_f32_crops: bad arguments"); return DM_E_INVALID;
    }
    if (reinterpret_cast<uintptr_t>(rects_dev) % 16) { set_error("dm_preprocess_patchify_f32_crops: rects must be 16-byte aligned (read as int4)"); return DM_E_INVALID; }
    cudaStream_t stream = (cudaStream_t)stream_;
    PreParams p;
    p.rgb = nullptr; p.H = Hi; p.W = Wi;
    const int rc = patchify_setup(p, B, net_h, net_w, patch, mean_host, std_host, chan_map_host, out, kpad, stream);
    if (rc) return rc;
    const long long total = (long long)B * net_h * net_w;
    preprocess_patchify_f32_crops_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p, img, Hi, Wi, rects_dev);
    DM_LAUNCH_CHECK("preprocess_patchify_f32_crops_kernel");
    return DM_OK;
}

DM_EXPORT int dm_assemble_tokens(const void *pe, const float *cls, const float *pos, float *X, int B, int Np, int C, void *stream_) {
    using namespace dm;
    if (C % 4) { set_error("dm_assemble_tokens: C must be a multiple of 4"); return DM_E_INVALID; }
    const long long total = (long long)B * (Np + 1) * (C / 4);
    assemble_tokens_kernel<__half><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)pe, cls, pos, X, B, Np, C);
    DM_LAUNCH_CHECK("assemble_tokens_kernel");
    return DM_OK;
}

/* the same with an fp32 patch embedding [B*Np, C] */
DM_EXPORT int dm_assemble_tokens_f32(const float *pe, const float *cls, const float *pos, float *X, int B, int Np, int C, void *stream_) {
    using namespace dm;
    if (C % 4) { set_error("dm_assemble_tokens_f32: C must be a multiple of 4"); return DM_E_INVALID; }
    const long long total = (long long)B * (Np + 1) * (C / 4);
    assemble_tokens_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(pe, cls, pos, X, B, Np, C);
    DM_LAUNCH_CHECK("assemble_tokens_kernel");
    return DM_OK;
}

DM_EXPORT int dm_layernorm_f16(const float *x, long long rows, int C, const float *gamma, const float *beta, float eps, void *out,
                               int tokens_per_img, int drop_first, void *stream_) {
    using namespace dm;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    switch (C) {
        case 384: layernorm_f16_kernel<3><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        case 768: layernorm_f16_kernel<6><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        case 1024: layernorm_f16_kernel<8><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        case 128: layernorm_f16_kernel<1><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        default: set_error("dm_layernorm_f16: unsupported width %d", C); return DM_E_UNSUPPORTED;
    }
    DM_LAUNCH_CHECK("layernorm_f16_kernel");
    return DM_OK;
}

DM_EXPORT int dm_layernorm_split(const float *x, long long rows, int C, const float *gamma, const float *beta, float eps, void *out,
                                 int tokens_per_img, int drop_first, void *stream_) {
    using namespace dm;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    switch (C) {
        case 384: layernorm_f16_kernel<3, true><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        case 768: layernorm_f16_kernel<6, true><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        case 1024: layernorm_f16_kernel<8, true><<<grid, 256, 0, stream>>>(x, rows, C, gamma, beta, eps, (__half *)out, tokens_per_img, drop_first); break;
        default: set_error("dm_layernorm_split: unsupported width %d", C); return DM_E_UNSUPPORTED;
    }
    DM_LAUNCH_CHECK("layernorm_f16_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_bilinear_nhwc_split(const void *in, int B, int Hin, int Win, int C, void *out, int Hout, int Wout, void *stream_) {
    using namespace dm;
    if (C % 4) { set_error("dm_resize_bilinear_nhwc_split: C must be a multiple of 4"); return DM_E_INVALID; }
    if (Hout > 65535 || B > 65535 || (long long)Hin * Win * 3 * C >= (1ll << 31) || (long long)Hout * Wout * 3 * C >= (1ll << 31)) {
        set_error("dm_resize_bilinear_nhwc_split: image too large for the 32-bit index path"); return DM_E_UNSUPPORTED;
    }
    const float sy = Hout > 1 ? (float)(Hin - 1) / (float)(Hout - 1) : 0.f;
    const float sx = Wout > 1 ? (float)(Win - 1) / (float)(Wout - 1) : 0.f;
    const dim3 grid((unsigned)((Wout * (C / 4) + 255) / 256), (unsigned)Hout, (unsigned)B);
    resize_bilinear_nhwc_split_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __half *)in, Hin, Win, C, (__half *)out, Hout, Wout, sy, sx);
    DM_LAUNCH_CHECK("resize_bilinear_nhwc_split_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_bilinear_nhwc_f16(const void *in, int B, int Hin, int Win, int C, void *out, int Hout, int Wout, void *stream_) {
    using namespace dm;
    if (C % 8) { set_error("dm_resize_bilinear_nhwc_f16: C must be a multiple of 8"); return DM_E_INVALID; }
    if (Hout > 65535 || B > 65535 || (long long)Hin * Win * C >= (1ll << 31) || (long long)Hout * Wout * C >= (1ll << 31)) {
        set_error("dm_resize_bilinear_nhwc_f16: image too large for the 32-bit index path"); return DM_E_UNSUPPORTED;
    }
    const float sy = Hout > 1 ? (float)(Hin - 1) / (float)(Hout - 1) : 0.f;
    const float sx = Wout > 1 ? (float)(Win - 1) / (float)(Wout - 1) : 0.f;
    const dim3 grid((unsigned)((Wout * (C / 8) + 255) / 256), (unsigned)Hout, (unsigned)B);
    resize_bilinear_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __half *)in, Hin, Win, C, (__half *)out, Hout, Wout, sy, sx);
    DM_LAUNCH_CHECK("resize_bilinear_nhwc_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_f32(const float *in, int B, int Hin, int Win, float *out, int Hout, int Wout, int mode, void *stream_) {
    using namespace dm;
    const long long total = (long long)B * Hout * Wout;
    resize_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(in, B, Hin, Win, out, Hout, Wout, mode, 1);
    DM_LAUNCH_CHECK("resize_f32_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_f32_ragged(const float *in, int B, int Hin, int Win, float *out, long long size, const dm_ragged_image *desc_host,
                                   const dm_ragged_image *desc_dev, int mode, void *stream_) {
    using namespace dm;
    int mh = 0, mw = 0;
    const int rc = check_ragged("dm_resize_f32_ragged", out, size, desc_host, desc_dev, B, 1, &mh, &mw);
    if (rc) return rc;
    if (!in || Hin <= 0 || Win <= 0 || (mode != 0 && mode != 1) || B > 65535) { set_error("dm_resize_f32_ragged: bad arguments"); return DM_E_INVALID; }
    const dim3 grid((unsigned)(((long long)mh * mw + 255) / 256), (unsigned)B);
    resize_f32_ragged_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>(in, Hin, Win, out, desc_dev, mode);
    DM_LAUNCH_CHECK("resize_f32_ragged_kernel");
    return DM_OK;
}

DM_EXPORT int dm_resize_f32_ld(const float *in, int ld, int B, int Hin, int Win, float *out, int Hout, int Wout, int mode, void *stream_) {
    using namespace dm;
    if (ld < 1) { set_error("dm_resize_f32_ld: bad pixel stride"); return DM_E_INVALID; }
    const long long total = (long long)B * Hout * Wout;
    resize_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(in, B, Hin, Win, out, Hout, Wout, mode, ld);
    DM_LAUNCH_CHECK("resize_f32_kernel");
    return DM_OK;
}

DM_EXPORT int dm_im2col_s2_f16(const void *in, int B, int H, int W, int C, void *out, void *stream_) {
    using namespace dm;
    if (C % 8) { set_error("dm_im2col_s2_f16: C must be a multiple of 8"); return DM_E_INVALID; }
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = (long long)B * Ho * Wo * 9 * (C / 8);
    im2col_s2_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)in, B, H, W, C, (__half *)out, Ho, Wo);
    DM_LAUNCH_CHECK("im2col_s2_kernel");
    return DM_OK;
}

DM_EXPORT int dm_im2col_s2_circular_f16(const void *in, int B, int H, int W, int C, void *out, void *stream_) {
    using namespace dm;
    if (!in || !out || B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8) { set_error("dm_im2col_s2_circular_f16: bad arguments (C must be a positive multiple of 8)"); return DM_E_INVALID; }
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = (long long)B * Ho * Wo * 9 * (C / 8);
    im2col_s2_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)in, B, H, W, C, (__half *)out, Ho, Wo);
    DM_LAUNCH_CHECK("im2col_s2_kernel");
    return DM_OK;
}

DM_EXPORT int dm_concat_readout_f16(const float *x, int B, int N, int C, void *out, void *stream_) {
    using namespace dm;
    if (C % 4) { set_error("dm_concat_readout_f16: C must be a multiple of 4"); return DM_E_INVALID; }
    if (N < 2 || (long long)B * (N - 1) >= (1ll << 31)) { set_error("dm_concat_readout_f16: bad token count"); return DM_E_INVALID; }
    concat_readout_kernel<<<(unsigned)(B * (N - 1)), 256, 0, (cudaStream_t)stream_>>>(x, B, N, C, (__half *)out);
    DM_LAUNCH_CHECK("concat_readout_kernel");
    return DM_OK;
}
