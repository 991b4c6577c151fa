// D8 — LeReS (ResNeXt-101 32x8d + FTB / FFM / AO decoder): the pieces that are not GEMMs or 3x3 stride-1 convolutions.
// Replaces parts of estimateleres / scale_torch (src/depthmap_generation.py:406-440), lib/Resnext_torch.py:196-220 and
// lib/network_auxi.py:95-215.  Everything else of the network runs on the wgmma GEMM / implicit-GEMM conv: 1x1 convs are GEMMs
// on NHWC activations, the 32-group 3x3 convs run as dense implicit GEMMs with block-diagonal filters (zero blocks between the
// groups keep the tensor core busy with exact zeros: 0.49 TFLOP-equivalent per 448^2 image instead of 0.29, but no new MMA shape),
// BatchNorm (inference statistics) is folded into the filters and biases at load time.
//   leres_stem_im2col   uint8 RGB -> /255 -> cv2.resize(bilinear) -> ImageNet normalise -> im2col of the 7x7 stride-2 pad-3 stem
//                       conv: fp16 [B*Ho*Wo, 192] (147 taps ordered (ky, kx, c), zero padded)
//   maxpool3x3s2_nhwc   F.max_pool2d(kernel 3, stride 2, padding 1) on fp16 NHWC
//   subsample2_nhwc     x[:, ::2, ::2, :]: the input of a stride-2 1x1 (downsample) convolution
//   add_f16             element-wise sum (FFM: ftb1(low) + high)
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace dm {

struct StemParams {
    const uint8_t *rgb;
    int B, H, W, nh, nw, Ho, Wo;
    float mean[3], inv_std[3];
    __half *out;     // [B*Ho*Wo, 192]
    const dm_ragged_image *ragged;      // ragged batch: image b is ragged[b] of the packed buffer rgb (H, W unused)
};

// cv2.resize INTER_LINEAR source coordinates of destination index d: sx, sx+1 (clamped) and the weight of sx+1
__device__ __forceinline__ void cv_linear_coord(int d, float scale, int n_src, int &i0, int &i1, float &f) {
    float fx = ((float)d + 0.5f) * scale - 0.5f;
    int sx = (int)floorf(fx);
    fx -= (float)sx;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= n_src - 1) { fx = 0.f; sx = n_src - 1; }
    i0 = sx; i1 = min(sx + 1, n_src - 1); f = fx;
}

// The 32 rows of a block (32 pixels x 8 ky-threads) are assembled in shared memory and leave as 16-byte stores: a thread's 21 values start at
// an odd 2-byte offset of the row, so direct stores would be 2 bytes each (the first version: 77 / 261 us for one 448^2 / 896^2 image).
__device__ __forceinline__ void stem_flush_rows(const __half *s_rows, __half *out, long long first_pix, long long total_pix) {
    const long long rows = min((long long)32, total_pix - first_pix);
    const uint4 *src = reinterpret_cast<const uint4 *>(s_rows);
    uint4 *dst = reinterpret_cast<uint4 *>(out + first_pix * 192);
    for (int i = threadIdx.x; i < (int)rows * 24; i += 256) dst[i] = src[i];
}

// CIRCULAR: the stem convolution's padding wraps around the network input (nn.Conv2d(padding_mode='circular')): a tap outside the
// net_h x net_w image samples the pixel net_h (net_w) rows (columns) away, before the resize maps it to the source
template <bool CIRCULAR>
__global__ void __launch_bounds__(256) leres_stem_im2col_kernel(StemParams p) {
    // one thread per (output pixel, ky): 7 kx taps x 3 channels = 21 values; thread ky == 7 zero-fills the 45 padding columns
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
        const int ox = (int)(pix % p.Wo), oy = (int)((pix / p.Wo) % p.Ho), b = (int)(pix / ((long long)p.Wo * p.Ho));
        const uint8_t *img = p.rgb + (long long)b * p.H * p.W * 3;
        const bool identity = p.nh == p.H && p.nw == p.W;           // cv2.resize to the same size is a copy
        const float sy = (float)p.H / (float)p.nh, sx = (float)p.W / (float)p.nw;
        const int iy = CIRCULAR ? wrap_index(oy * 2 - 3 + ky, p.nh) : oy * 2 - 3 + ky;
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = CIRCULAR ? wrap_index(ox * 2 - 3 + kx, p.nw) : ox * 2 - 3 + kx;
            float v[3] = {0.f, 0.f, 0.f};
            if (iy >= 0 && iy < p.nh && ix >= 0 && ix < p.nw) {
                if (identity) {
                    const uint8_t *px = img + ((long long)iy * p.W + ix) * 3;
                    v[0] = (float)px[0] / 255.f; v[1] = (float)px[1] / 255.f; v[2] = (float)px[2] / 255.f;
                } else {
                    int y0, y1, x0, x1; float fy, fx;
                    cv_linear_coord(iy, sy, p.H, y0, y1, fy);
                    cv_linear_coord(ix, sx, p.W, x0, x1, fx);
                    const uint8_t *p00 = img + ((long long)y0 * p.W + x0) * 3, *p01 = img + ((long long)y0 * p.W + x1) * 3;
                    const uint8_t *p10 = img + ((long long)y1 * p.W + x0) * 3, *p11 = img + ((long long)y1 * p.W + x1) * 3;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float a = ((float)p00[c] * (1.f - fx) + (float)p01[c] * fx) / 255.f, d = ((float)p10[c] * (1.f - fx) + (float)p11[c] * fx) / 255.f;
                        v[c] = a * (1.f - fy) + d * fy;
                    }
                }
                // the network sees RGB in source order (the holder's channel swap is undone by estimateleres, :408); ImageNet statistics
#pragma unroll
                for (int c = 0; c < 3; ++c) v[c] = (v[c] - p.mean[c]) * p.inv_std[c];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) row[(ky * 7 + kx) * 3 + c] = __float2half_rn(v[c]);
        }
    }
    __syncthreads();
    stem_flush_rows(s_rows, p.out, (long long)blockIdx.x * 32, total_pix);
}

// ragged twin of leres_stem_im2col_kernel: image b is p.ragged[b] of the packed buffer p.rgb
template <bool CIRCULAR>
__global__ void __launch_bounds__(256) leres_stem_im2col_ragged_kernel(StemParams p) {
    // one thread per (output pixel, ky): 7 kx taps x 3 channels = 21 values; thread ky == 7 zero-fills the 45 padding columns
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
        const int ox = (int)(pix % p.Wo), oy = (int)((pix / p.Wo) % p.Ho), b = (int)(pix / ((long long)p.Wo * p.Ho));
        const dm_ragged_image d = p.ragged[b];
        const uint8_t *img = p.rgb + d.offset;
        const int H = d.h, W = d.w;
        const bool identity = p.nh == H && p.nw == W;           // cv2.resize to the same size is a copy
        const float sy = (float)H / (float)p.nh, sx = (float)W / (float)p.nw;
        const int iy = CIRCULAR ? wrap_index(oy * 2 - 3 + ky, p.nh) : oy * 2 - 3 + ky;
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = CIRCULAR ? wrap_index(ox * 2 - 3 + kx, p.nw) : ox * 2 - 3 + kx;
            float v[3] = {0.f, 0.f, 0.f};
            if (iy >= 0 && iy < p.nh && ix >= 0 && ix < p.nw) {
                if (identity) {
                    const uint8_t *px = img + ((long long)iy * W + ix) * 3;
                    v[0] = (float)px[0] / 255.f; v[1] = (float)px[1] / 255.f; v[2] = (float)px[2] / 255.f;
                } else {
                    int y0, y1, x0, x1; float fy, fx;
                    cv_linear_coord(iy, sy, H, y0, y1, fy);
                    cv_linear_coord(ix, sx, W, x0, x1, fx);
                    const uint8_t *p00 = img + ((long long)y0 * W + x0) * 3, *p01 = img + ((long long)y0 * W + x1) * 3;
                    const uint8_t *p10 = img + ((long long)y1 * W + x0) * 3, *p11 = img + ((long long)y1 * W + x1) * 3;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float a = ((float)p00[c] * (1.f - fx) + (float)p01[c] * fx) / 255.f, d = ((float)p10[c] * (1.f - fx) + (float)p11[c] * fx) / 255.f;
                        v[c] = a * (1.f - fy) + d * fy;
                    }
                }
                // the network sees RGB in source order (the holder's channel swap is undone by estimateleres, :408); ImageNet statistics
#pragma unroll
                for (int c = 0; c < 3; ++c) v[c] = (v[c] - p.mean[c]) * p.inv_std[c];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) row[(ky * 7 + kx) * 3 + c] = __float2half_rn(v[c]);
        }
    }
    __syncthreads();
    stem_flush_rows(s_rows, p.out, (long long)blockIdx.x * 32, total_pix);
}

__global__ void __launch_bounds__(256) maxpool3x3s2_nhwc_kernel(const __half *__restrict__ in, int H, int W, int C, __half *__restrict__ out, int Ho, int Wo) {
    const int c8 = C >> 3;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= Wo * c8) return;
    const int x = t / c8, c = (t - x * c8) << 3;
    const int y = blockIdx.y, b = blockIdx.z;
    float m[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) m[k] = -INFINITY;
    for (int dy = 0; dy < 3; ++dy) {
        const int iy = 2 * y - 1 + dy;
        if (iy < 0 || iy >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int ix = 2 * x - 1 + dx;
            if (ix < 0 || ix >= W) continue;
            const uint4 u = __ldg(reinterpret_cast<const uint4 *>(in + (((size_t)b * H + iy) * W + ix) * C + c));
            const __half2 *h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
            for (int k = 0; k < 4; ++k) { const float2 f = __half22float2(h[k]); m[2 * k] = fmaxf(m[2 * k], f.x); m[2 * k + 1] = fmaxf(m[2 * k + 1], f.y); }
        }
    }
    uint4 o;
    __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(m[2 * k], m[2 * k + 1]);
    *reinterpret_cast<uint4 *>(out + (((size_t)b * Ho + y) * Wo + x) * C + c) = o;
}

__global__ void __launch_bounds__(256) subsample2_nhwc_kernel(const __half *__restrict__ in, int H, int W, int C, __half *__restrict__ out, int Ho, int Wo) {
    const int c8 = C >> 3;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= Wo * c8) return;
    const int x = t / c8, c = (t - x * c8) << 3;
    const int y = blockIdx.y, b = blockIdx.z;
    *reinterpret_cast<uint4 *>(out + (((size_t)b * Ho + y) * Wo + x) * C + c) =
        __ldg(reinterpret_cast<const uint4 *>(in + (((size_t)b * H + 2 * y) * W + 2 * x) * C + c));
}

__global__ void __launch_bounds__(256) add_f16_kernel(const __half *__restrict__ a, const __half *__restrict__ b, __half *__restrict__ out, long long n8) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const uint4 ua = __ldg(reinterpret_cast<const uint4 *>(a) + i), ub = __ldg(reinterpret_cast<const uint4 *>(b) + i);
    const __half2 *ha = reinterpret_cast<const __half2 *>(&ua), *hb = reinterpret_cast<const __half2 *>(&ub);
    uint4 o;
    __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float2 x = __half22float2(ha[k]), y = __half22float2(hb[k]); oh[k] = __floats2half2_rn(x.x + y.x, x.y + y.y); }
    reinterpret_cast<uint4 *>(out)[i] = o;
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

template <bool CIRCULAR>
static int leres_stem_im2col(const char *who, const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host,
                             const float *std_host, void *out, void *stream_) {
    using namespace dm;
    if (!rgb || !out || B <= 0 || net_h <= 0 || net_w <= 0) { set_error("%s: bad arguments", who); return DM_E_INVALID; }
    StemParams p;
    p.rgb = rgb; p.B = B; p.H = H; p.W = W; p.nh = net_h; p.nw = net_w;
    p.Ho = (net_h + 6 - 7) / 2 + 1; p.Wo = (net_w + 6 - 7) / 2 + 1;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; }
    p.out = (__half *)out;
    const long long total = (long long)B * p.Ho * p.Wo * 8;
    leres_stem_im2col_kernel<CIRCULAR><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("leres_stem_im2col_kernel");
    return DM_OK;
}

DM_EXPORT int dm_leres_stem_im2col(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host, const float *std_host,
                                   void *out, void *stream_) {
    return leres_stem_im2col<false>("dm_leres_stem_im2col", rgb, B, H, W, net_h, net_w, mean_host, std_host, out, stream_);
}

DM_EXPORT int dm_leres_stem_im2col_circular(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host,
                                            const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col<true>("dm_leres_stem_im2col_circular", rgb, B, H, W, net_h, net_w, mean_host, std_host, out, stream_);
}

template <bool CIRCULAR>
static int leres_stem_im2col_ragged(const char *who, const uint8_t *packed, long long size, const dm_ragged_image *desc_host,
                                    const dm_ragged_image *desc_dev, int B, int net_h, int net_w, const float *mean_host, const float *std_host,
                                    void *out, void *stream_) {
    using namespace dm;
    const int rc = check_ragged(who, packed, size, desc_host, desc_dev, B, 3, nullptr, nullptr);
    if (rc) return rc;
    if (!out || !mean_host || !std_host || net_h <= 0 || net_w <= 0) { set_error("%s: bad arguments", who); return DM_E_INVALID; }
    StemParams p;
    p.rgb = packed; p.ragged = desc_dev; p.B = B; p.H = 0; p.W = 0; p.nh = net_h; p.nw = net_w;
    p.Ho = (net_h + 6 - 7) / 2 + 1; p.Wo = (net_w + 6 - 7) / 2 + 1;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; }
    p.out = (__half *)out;
    const long long total = (long long)B * p.Ho * p.Wo * 8;
    leres_stem_im2col_ragged_kernel<CIRCULAR><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("leres_stem_im2col_ragged_kernel");
    return DM_OK;
}

DM_EXPORT int dm_leres_stem_im2col_ragged(const uint8_t *packed, long long size, const dm_ragged_image *desc_host, const dm_ragged_image *desc_dev,
                                          int B, int net_h, int net_w, const float *mean_host, const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_ragged<false>("dm_leres_stem_im2col_ragged", packed, size, desc_host, desc_dev, B, net_h, net_w, mean_host, std_host,
                                           out, stream_);
}

DM_EXPORT int dm_leres_stem_im2col_ragged_circular(const uint8_t *packed, long long size, const dm_ragged_image *desc_host,
                                                   const dm_ragged_image *desc_dev, int B, int net_h, int net_w, const float *mean_host,
                                                   const float *std_host, void *out, void *stream_) {
    return leres_stem_im2col_ragged<true>("dm_leres_stem_im2col_ragged_circular", packed, size, desc_host, desc_dev, B, net_h, net_w, mean_host,
                                          std_host, out, stream_);
}

DM_EXPORT int dm_maxpool3x3s2_nhwc_f16(const void *in, int B, int H, int W, int C, void *out, void *stream_) {
    using namespace dm;
    if (C % 8) { set_error("dm_maxpool3x3s2_nhwc_f16: C must be a multiple of 8"); return DM_E_INVALID; }
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    if (Ho > 65535 || B > 65535) { set_error("dm_maxpool3x3s2_nhwc_f16: shape too large"); return DM_E_UNSUPPORTED; }
    maxpool3x3s2_nhwc_kernel<<<dim3((unsigned)((Wo * (C / 8) + 255) / 256), Ho, B), 256, 0, (cudaStream_t)stream_>>>((const __half *)in, H, W, C, (__half *)out, Ho, Wo);
    DM_LAUNCH_CHECK("maxpool3x3s2_nhwc_kernel");
    return DM_OK;
}

DM_EXPORT int dm_subsample2_nhwc_f16(const void *in, int B, int H, int W, int C, void *out, void *stream_) {
    using namespace dm;
    if (C % 8) { set_error("dm_subsample2_nhwc_f16: C must be a multiple of 8"); return DM_E_INVALID; }
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    if (Ho > 65535 || B > 65535) { set_error("dm_subsample2_nhwc_f16: shape too large"); return DM_E_UNSUPPORTED; }
    subsample2_nhwc_kernel<<<dim3((unsigned)((Wo * (C / 8) + 255) / 256), Ho, B), 256, 0, (cudaStream_t)stream_>>>((const __half *)in, H, W, C, (__half *)out, Ho, Wo);
    DM_LAUNCH_CHECK("subsample2_nhwc_kernel");
    return DM_OK;
}

DM_EXPORT int dm_add_f16(const void *a, const void *b, void *out, long long n, void *stream_) {
    using namespace dm;
    if (n % 8) { set_error("dm_add_f16: element count must be a multiple of 8"); return DM_E_INVALID; }
    add_f16_kernel<<<(unsigned)((n / 8 + 255) / 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)a, (const __half *)b, (__half *)out, n / 8);
    DM_LAUNCH_CHECK("add_f16_kernel");
    return DM_OK;
}
