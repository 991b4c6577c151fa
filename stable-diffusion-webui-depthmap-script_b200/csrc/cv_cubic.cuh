// cv2.resize(..., INTER_CUBIC) sampling shared by the patchify kernels (vit_kernels.cu) and the MidasNet stem (midas_kernels.cu):
// separable, A = -0.75, replicated borders, float coefficients.
#pragma once
#include <stdint.h>

namespace dm {

__device__ __forceinline__ void cubic_coeffs(float x, float *c) {
    const float A = -0.75f;
    c[0] = ((A * (x + 1.f) - 5.f * A) * (x + 1.f) + 8.f * A) * (x + 1.f) - 4.f * A;
    c[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
    c[2] = ((A + 2.f) * (1.f - x) - (A + 3.f)) * (1.f - x) * (1.f - x) + 1.f;
    c[3] = 1.f - c[0] - c[1] - c[2];
}

// Pixel sources: load(y, x, v) reads the three channels of source pixel (y, x) as floats.
struct U8Source {               // one image of a uint8 [B, H, W, 3] batch
    const uint8_t *img;
    int H, W;
    __device__ __forceinline__ void load(int y, int x, float (&v)[3]) const {
        const uint8_t *px = img + ((long long)y * W + x) * 3;
        v[0] = px[0]; v[1] = px[1]; v[2] = px[2];
    }
};
struct F32CropSource {          // a (x0, y0, w, h) crop of a planar fp32 [3, Hi, Wi] image
    const float *img;
    long long plane;
    int pitch, H, W;
    __device__ __forceinline__ void load(int y, int x, float (&v)[3]) const {
        const float *px = img + (long long)y * pitch + x;
        v[0] = px[0]; v[1] = px[plane]; v[2] = px[2 * plane];
    }
};

// network pixel (y, x) of an nh x nw input: the source pixel when the sizes match, otherwise cv2.resize(..., INTER_CUBIC)
template <class Src>
__device__ __forceinline__ void cubic_sample(const Src &src, int nh, int nw, int y, int x, float (&v)[3]) {
    if (nh == src.H && nw == src.W) { src.load(y, x, v); return; }
    const float sx = (float)src.W / (float)nw, sy = (float)src.H / (float)nh;
    float fx = ((float)x + 0.5f) * sx - 0.5f, fy = ((float)y + 0.5f) * sy - 0.5f;
    const int ix = (int)floorf(fx), iy = (int)floorf(fy);
    fx -= (float)ix; fy -= (float)iy;
    float cx[4], cy[4];
    cubic_coeffs(fx, cx);
    cubic_coeffs(fy, cy);
    v[0] = v[1] = v[2] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int yy = min(max(iy - 1 + j, 0), src.H - 1);
        float r[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int xx = min(max(ix - 1 + i, 0), src.W - 1);
            float px[3];
            src.load(yy, xx, px);
            r[0] = fmaf(cx[i], px[0], r[0]); r[1] = fmaf(cx[i], px[1], r[1]); r[2] = fmaf(cx[i], px[2], r[2]);
        }
        v[0] = fmaf(cy[j], r[0], v[0]); v[1] = fmaf(cy[j], r[1], v[1]); v[2] = fmaf(cy[j], r[2], v[2]);
    }
}

}  // namespace dm
