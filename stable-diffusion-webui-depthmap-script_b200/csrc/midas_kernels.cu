// MiDaS v2.1 (MidasNet, model type 5): the pieces its ResNeXt-101 encoder and RefineNet decoder need beyond the LeReS kernels.
// Replaces parts of estimatemidas (src/depthmap_generation.py:455-499, dmidas/transforms.py:48-231) and dmidas/midas_net.py:47-76.
//   midas_stem_im2col          uint8 RGB -> cv2.resize(INTER_CUBIC) -> /255 -> ImageNet normalise -> channel map -> im2col of the
//                              7x7 stride-2 pad-3 stem conv: fp16 [B*Ho*Wo, 192], the layout of leres_stem_im2col (147 taps
//                              ordered (ky, kx, c), zero padded), so the same stem GEMM consumes it
//   midas_stem_im2col_f32_crops  the same for B crops of one planar fp32 image (BOOST's estimatemidasBoost: no /255)
//   resize_bilinear_half_nhwc  fp16 NHWC bilinear, align_corners=False (the head's Interpolate, dmidas/blocks.py:202-227)
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "cv_cubic.cuh"

namespace dm {

struct MidasStemParams {
    const uint8_t *rgb;     // [B, H, W, 3] (uint8 variant)
    const float *img;       // [3, Hi, Wi] planar image (crop variant)
    const int *rects;       // [B][4] = x0, y0, w, h (crop variant)
    long long plane;
    int B, H, W, nh, nw, Ho, Wo;
    float value_scale, mean[3], inv_std[3];
    int chan_map[3];        // network channel c reads source channel chan_map[c]
    __half *out;            // [B*Ho*Wo, 192]
    const dm_ragged_image *ragged;      // RAGGED (uint8 variant): image b is ragged[b] of the packed buffer rgb (H, W unused)
};

// One thread per (output pixel, ky): 7 kx taps x 3 channels, each tap a 4x4 cubic sample of the source (L1 / L2 hits: a network
// pixel is read by ~12 taps).  Thread ky == 7 zero-fills the 45 padding columns.  The 32 rows of a block are assembled in shared
// memory and leave as 16-byte stores, as in leres_stem_im2col.  CIRCULAR: a tap outside the nh x nw network input wraps around
// (nn.Conv2d(padding_mode='circular')) before the resize maps it to the source.
template <bool F32, bool CIRCULAR, bool RAGGED = false>
__global__ void __launch_bounds__(256) midas_stem_im2col_kernel(MidasStemParams p) {
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
        U8Source u8{nullptr, p.H, p.W};
        F32CropSource f32{nullptr, p.plane, p.W, p.H, p.W};
        if (F32) {
            const int4 r = __ldg(reinterpret_cast<const int4 *>(p.rects) + b);
            f32 = F32CropSource{p.img + (long long)r.y * p.W + r.x, p.plane, p.W, r.w, r.z};
        } else if (RAGGED) {
            const dm_ragged_image d = p.ragged[b];
            u8 = U8Source{p.rgb + d.offset, d.h, d.w};
        } else {
            u8.img = p.rgb + (long long)b * p.H * p.W * 3;
        }
        const int iy = CIRCULAR ? wrap_index(oy * 2 - 3 + ky, p.nh) : oy * 2 - 3 + ky;
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = CIRCULAR ? wrap_index(ox * 2 - 3 + kx, p.nw) : ox * 2 - 3 + kx;
            float o[3] = {0.f, 0.f, 0.f};
            if (iy >= 0 && iy < p.nh && ix >= 0 && ix < p.nw) {
                float v[3];
                if (F32) cubic_sample(f32, p.nh, p.nw, iy, ix, v);
                else cubic_sample(u8, p.nh, p.nw, iy, ix, v);
#pragma unroll
                for (int c = 0; c < 3; ++c) {     // selects, not v[chan_map[c]]: a dynamic index would put v in local memory
                    const float s = p.chan_map[c] == 0 ? v[0] : (p.chan_map[c] == 1 ? v[1] : v[2]);
                    o[c] = (s * p.value_scale - p.mean[c]) * p.inv_std[c];
                }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) row[(ky * 7 + kx) * 3 + c] = __float2half_rn(o[c]);
        }
    }
    __syncthreads();
    const long long first = (long long)blockIdx.x * 32;
    const long long rows = min((long long)32, total_pix - first);
    const uint4 *src = reinterpret_cast<const uint4 *>(s_rows);
    uint4 *dst = reinterpret_cast<uint4 *>(p.out + first * 192);
    for (int i = threadIdx.x; i < (int)rows * 24; i += 256) dst[i] = src[i];
}

// torch upsample_bilinear2d, align_corners=False: source coordinate (d + 0.5) * in / out - 0.5, clamped at 0; one thread per
// (output pixel, 8 channels), the grid layout of resize_bilinear_nhwc_kernel (vit_kernels.cu)
__global__ void __launch_bounds__(256) resize_bilinear_half_nhwc_kernel(const __half *__restrict__ in, int Hin, int Win, int C,
                                                                        __half *__restrict__ out, int Hout, int Wout, float sy, float sx) {
    const int c8 = C >> 3;
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= Wout * c8) return;
    const int x = t / c8;
    const int c = (t - x * c8) << 3;
    const int y = blockIdx.y, b = blockIdx.z;
    const float fy = fmaxf(sy * ((float)y + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * ((float)x + 0.5f) - 0.5f, 0.f);
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
        const float r0 = hy * (hx * f00.x + lx * f01.x) + ly * (hx * f10.x + lx * f11.x);
        const float r1 = hy * (hx * f00.y + lx * f01.y) + ly * (hx * f10.y + lx * f11.y);
        oh[k] = __floats2half2_rn(r0, r1);
    }
    __stcs(reinterpret_cast<uint4 *>(out + ((size_t)(b * Hout + y) * Wout + x) * C + c), o);
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

template <bool F32, bool CIRCULAR, bool RAGGED = false>
static int midas_stem_im2col(const char *who, dm::MidasStemParams &p, int net_h, int net_w, const float *mean_host, const float *std_host,
                             const int *chan_map_host, void *out, void *stream_) {
    using namespace dm;
    if (!out || !mean_host || !std_host || !chan_map_host || p.B <= 0 || p.H <= 0 || p.W <= 0 || net_h <= 0 || net_w <= 0) {
        set_error("%s: bad arguments", who); return DM_E_INVALID;
    }
    for (int c = 0; c < 3; ++c) {
        if (chan_map_host[c] < 0 || chan_map_host[c] > 2) { set_error("%s: channel map entries must be 0, 1 or 2", who); return DM_E_INVALID; }
        p.mean[c] = mean_host[c]; p.inv_std[c] = 1.0f / std_host[c]; p.chan_map[c] = chan_map_host[c];
    }
    p.nh = net_h; p.nw = net_w;
    p.Ho = (net_h + 6 - 7) / 2 + 1; p.Wo = (net_w + 6 - 7) / 2 + 1;
    p.out = (__half *)out;
    const long long total = (long long)p.B * p.Ho * p.Wo * 8;
    midas_stem_im2col_kernel<F32, CIRCULAR, RAGGED><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(p);
    DM_LAUNCH_CHECK("midas_stem_im2col_kernel");
    return DM_OK;
}

template <bool CIRCULAR>
static int midas_stem_u8(const char *who, const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host,
                         const float *std_host, const int *chan_map_host, void *out, void *stream_) {
    if (!rgb) { dm::set_error("%s: rgb is NULL", who); return DM_E_INVALID; }
    dm::MidasStemParams p{};
    p.rgb = rgb; p.B = B; p.H = H; p.W = W; p.value_scale = 1.0f / 255.0f;
    return midas_stem_im2col<false, CIRCULAR>(who, p, net_h, net_w, mean_host, std_host, chan_map_host, out, stream_);
}

template <bool CIRCULAR>
static int midas_stem_crops(const char *who, const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w,
                            const float *mean_host, const float *std_host, const int *chan_map_host, void *out, void *stream_) {
    if (!img || !rects_dev) { dm::set_error("%s: null argument", who); return DM_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(rects_dev) % 16) { dm::set_error("%s: rects must be 16-byte aligned (read as int4)", who); return DM_E_INVALID; }
    dm::MidasStemParams p{};
    p.img = img; p.rects = rects_dev; p.plane = (long long)Hi * Wi; p.B = B; p.H = Hi; p.W = Wi; p.value_scale = 1.0f;
    return midas_stem_im2col<true, CIRCULAR>(who, p, net_h, net_w, mean_host, std_host, chan_map_host, out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host, const float *std_host,
                                   const int *chan_map_host, void *out, void *stream_) {
    return midas_stem_u8<false>("dm_midas_stem_im2col", rgb, B, H, W, net_h, net_w, mean_host, std_host, chan_map_host, out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col_circular(const uint8_t *rgb, int B, int H, int W, int net_h, int net_w, const float *mean_host,
                                            const float *std_host, const int *chan_map_host, void *out, void *stream_) {
    return midas_stem_u8<true>("dm_midas_stem_im2col_circular", rgb, B, H, W, net_h, net_w, mean_host, std_host, chan_map_host, out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col_f32_crops(const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w,
                                             const float *mean_host, const float *std_host, const int *chan_map_host, void *out, void *stream_) {
    return midas_stem_crops<false>("dm_midas_stem_im2col_f32_crops", img, Hi, Wi, rects_dev, B, net_h, net_w, mean_host, std_host, chan_map_host,
                                   out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col_f32_crops_circular(const float *img, int Hi, int Wi, const int *rects_dev, int B, int net_h, int net_w,
                                                      const float *mean_host, const float *std_host, const int *chan_map_host, void *out,
                                                      void *stream_) {
    return midas_stem_crops<true>("dm_midas_stem_im2col_f32_crops_circular", img, Hi, Wi, rects_dev, B, net_h, net_w, mean_host, std_host,
                                  chan_map_host, out, stream_);
}

template <bool CIRCULAR>
static int midas_stem_ragged(const char *who, const uint8_t *packed, long long size, const dm_ragged_image *desc_host,
                             const dm_ragged_image *desc_dev, int B, int net_h, int net_w, const float *mean_host, const float *std_host,
                             const int *chan_map_host, void *out, void *stream_) {
    int mh = 0, mw = 0;
    const int rc = dm::check_ragged(who, packed, size, desc_host, desc_dev, B, 3, &mh, &mw);
    if (rc) return rc;
    dm::MidasStemParams p{};
    p.rgb = packed; p.ragged = desc_dev; p.B = B; p.H = mh; p.W = mw; p.value_scale = 1.0f / 255.0f;    // H, W: only checked > 0
    return midas_stem_im2col<false, CIRCULAR, true>(who, p, net_h, net_w, mean_host, std_host, chan_map_host, out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col_ragged(const uint8_t *packed, long long size, const dm_ragged_image *desc_host, const dm_ragged_image *desc_dev,
                                          int B, int net_h, int net_w, const float *mean_host, const float *std_host, const int *chan_map_host,
                                          void *out, void *stream_) {
    return midas_stem_ragged<false>("dm_midas_stem_im2col_ragged", packed, size, desc_host, desc_dev, B, net_h, net_w, mean_host, std_host,
                                    chan_map_host, out, stream_);
}

DM_EXPORT int dm_midas_stem_im2col_ragged_circular(const uint8_t *packed, long long size, const dm_ragged_image *desc_host,
                                                   const dm_ragged_image *desc_dev, int B, int net_h, int net_w, const float *mean_host,
                                                   const float *std_host, const int *chan_map_host, void *out, void *stream_) {
    return midas_stem_ragged<true>("dm_midas_stem_im2col_ragged_circular", packed, size, desc_host, desc_dev, B, net_h, net_w, mean_host,
                                   std_host, chan_map_host, out, stream_);
}

DM_EXPORT int dm_resize_bilinear_half_nhwc_f16(const void *in, int B, int Hin, int Win, int C, void *out, int Hout, int Wout, void *stream_) {
    using namespace dm;
    if (!in || !out || B <= 0 || Hin <= 0 || Win <= 0 || Hout <= 0 || Wout <= 0 || C <= 0 || C % 8) {
        set_error("dm_resize_bilinear_half_nhwc_f16: bad arguments (C must be a positive multiple of 8)"); return DM_E_INVALID;
    }
    if (Hout > 65535 || B > 65535 || (long long)Hin * Win * C >= (1ll << 31) || (long long)Hout * Wout * C >= (1ll << 31)) {
        set_error("dm_resize_bilinear_half_nhwc_f16: image too large for the 32-bit index path"); return DM_E_UNSUPPORTED;
    }
    const dim3 grid((unsigned)((Wout * (C / 8) + 255) / 256), (unsigned)Hout, (unsigned)B);
    resize_bilinear_half_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __half *)in, Hin, Win, C, (__half *)out, Hout, Wout,
                                                                              (float)Hin / (float)Hout, (float)Win / (float)Wout);
    DM_LAUNCH_CHECK("resize_bilinear_half_nhwc_kernel");
    return DM_OK;
}
