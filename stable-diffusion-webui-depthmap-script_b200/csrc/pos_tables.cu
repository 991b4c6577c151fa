// Resolution-dependent tables of the ViT trunks, host arithmetic in float32 and in torch's operation order, so that the
// engines (depthmap_generation.py) feed the kernels bit-for-bit the numbers the reference's torch code computes:
//   dm_dinov2_pos_embed  DINOv2 interpolate_pos_encoding (dinov2.py:179-210)
//   dm_vit_pos_embed     MiDaS 3.0 _resize_pos_embed (dmidas/backbones/vit.py:16-31)
//   dm_beit_rel_table    BEiT _get_rel_pos_bias, table half (dmidas/backbones/beit.py:29-50)
// They run once per resolution; the engines cache the results on the device.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace dm {

// torch upsample_bilinear2d, align_corners=False: src = max((dst + 0.5) * in/out - 0.5, 0), float32 arithmetic
static void bilinear_table(const float *src, int ih, int iw, float *dst, int oh, int ow) {
    const float sy = (float)ih / (float)oh, sx = (float)iw / (float)ow;
    for (int y = 0; y < oh; ++y) {
        float fy = sy * ((float)y + 0.5f) - 0.5f; if (fy < 0.f) fy = 0.f;
        const int y0 = (int)fy, y1 = y0 + (y0 < ih - 1 ? 1 : 0);
        const float ly = fy - (float)y0, hy = 1.f - ly;
        for (int x = 0; x < ow; ++x) {
            float fx = sx * ((float)x + 0.5f) - 0.5f; if (fx < 0.f) fx = 0.f;
            const int x0 = (int)fx, x1 = x0 + (x0 < iw - 1 ? 1 : 0);
            const float lx = fx - (float)x0, hx = 1.f - lx;
            dst[y * ow + x] = hy * (hx * src[y0 * iw + x0] + lx * src[y0 * iw + x1]) + ly * (hx * src[y1 * iw + x0] + lx * src[y1 * iw + x1]);
        }
    }
}

// BEiT: the [nrd0, heads] table of one block resized to the current window (dmidas/backbones/beit.py:29-50), laid out
// [heads, nrd] and multiplied by log2(e).  Host arithmetic, float32, in torch's operation order.
static void beit_rel_table_host(const float *t, int window, int heads, int gh, int gw, float *out) {
    const int old = 2 * window - 1, nh = 2 * gh - 1, nw = 2 * gw - 1, nrd = nh * nw + 3;
    std::vector<float> plane((size_t)old * old), res((size_t)nh * nw);
    for (int hd = 0; hd < heads; ++hd) {
        // sub = table[:old*old].reshape(1, old_w, old_h, heads).permute(0, 3, 1, 2): plane[a][b] = table[a*old + b][hd]
        for (int a = 0; a < old * old; ++a) plane[a] = t[(size_t)a * heads + hd];
        if (nh == old && nw == old) res = plane; else bilinear_table(plane.data(), old, old, res.data(), nh, nw);
        for (int a = 0; a < nh * nw; ++a) out[(size_t)hd * nrd + a] = res[a] * 1.4426950408889634f;
        for (int e = 0; e < 3; ++e) out[(size_t)hd * nrd + nh * nw + e] = t[(size_t)(old * old + e) * heads + hd] * 1.4426950408889634f;
    }
}

// DINOv2 interpolate_pos_encoding (dinov2.py:179-210): bicubic (A = -0.75, align_corners=False) with scale factors
// (gh + 0.1) / n, (gw + 0.1) / n; identity for the native square grid.  torch uses 1/scale_factor as the coordinate scale.
static void cubic_w(float x, float *c) {
    const float A = -0.75f;
    c[0] = ((A * (x + 1.f) - 5.f * A) * (x + 1.f) + 8.f * A) * (x + 1.f) - 4.f * A;
    c[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
    c[2] = ((A + 2.f) * (1.f - x) - (A + 3.f)) * (1.f - x) * (1.f - x) + 1.f;
    c[3] = ((A * (2.f - x) - 5.f * A) * (2.f - x) + 8.f * A) * (2.f - x) - 4.f * A;
}
// MiDaS 3.0 _resize_pos_embed (dmidas/backbones/vit.py:16-31): class entry kept, the n x n grid resized bilinearly
// (align_corners=False) to gh x gw
static void vit_pos_embed_host(const float *pe, int n, int C, int gh, int gw, float *out) {
    for (int k = 0; k < C; ++k) out[k] = pe[k];
    if (gh == n && gw == n) { memcpy(out + C, pe + C, (size_t)n * n * C * sizeof(float)); return; }
    std::vector<float> plane((size_t)n * n), res((size_t)gh * gw);
    for (int k = 0; k < C; ++k) {
        for (int a = 0; a < n * n; ++a) plane[a] = pe[(size_t)(1 + a) * C + k];
        bilinear_table(plane.data(), n, n, res.data(), gh, gw);
        for (int a = 0; a < gh * gw; ++a) out[(size_t)(1 + a) * C + k] = res[a];
    }
}

static void dinov2_pos_embed_host(const float *pe, int n, int C, int gh, int gw, float *out) {
    for (int k = 0; k < C; ++k) out[k] = pe[k];
    if (gh == n && gw == n) {
        memcpy(out + C, pe + C, (size_t)n * n * C * sizeof(float));
        return;
    }
    // the reference hands (w, h) = (tensor H, tensor W) to the function, so the FIRST spatial axis of the n x n grid follows gh
    const double sf_y = ((double)gh + 0.1) / sqrt((double)(n * n)), sf_x = ((double)gw + 0.1) / sqrt((double)(n * n));
    const float sy = (float)(1.0 / sf_y), sx = (float)(1.0 / sf_x);
    for (int y = 0; y < gh; ++y) {
        const float fy = sy * ((float)y + 0.5f) - 0.5f;
        const int iy = (int)floorf(fy);
        float cy[4]; cubic_w(fy - (float)iy, cy);
        for (int x = 0; x < gw; ++x) {
            const float fx = sx * ((float)x + 0.5f) - 0.5f;
            const int ix = (int)floorf(fx);
            float cx[4]; cubic_w(fx - (float)ix, cx);
            float *o = out + (size_t)(1 + y * gw + x) * C;
            for (int k = 0; k < C; ++k) o[k] = 0.f;
            for (int j = 0; j < 4; ++j) {
                const int yy = std::min(std::max(iy - 1 + j, 0), n - 1);
                for (int i = 0; i < 4; ++i) {
                    const int xx = std::min(std::max(ix - 1 + i, 0), n - 1);
                    const float wgt = cy[j] * cx[i];
                    const float *s = pe + (size_t)(1 + yy * n + xx) * C;
                    for (int k = 0; k < C; ++k) o[k] += wgt * s[k];
                }
            }
        }
    }
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

DM_EXPORT int dm_dinov2_pos_embed(const float *pos_embed_host, int n, int C, int gh, int gw, float *out_host) {
    if (!pos_embed_host || !out_host || n <= 0 || C <= 0 || gh <= 0 || gw <= 0) { dm::set_error("dm_dinov2_pos_embed: bad arguments"); return DM_E_INVALID; }
    dm::dinov2_pos_embed_host(pos_embed_host, n, C, gh, gw, out_host);
    return DM_OK;
}
DM_EXPORT int dm_vit_pos_embed(const float *pos_embed_host, int n, int C, int gh, int gw, float *out_host) {
    if (!pos_embed_host || !out_host || n <= 0 || C <= 0 || gh <= 0 || gw <= 0) { dm::set_error("dm_vit_pos_embed: bad arguments"); return DM_E_INVALID; }
    dm::vit_pos_embed_host(pos_embed_host, n, C, gh, gw, out_host);
    return DM_OK;
}
DM_EXPORT int dm_beit_rel_table(const float *table_host, int window, int heads, int gh, int gw, float *out_host) {
    if (!table_host || !out_host || window <= 0 || heads <= 0 || gh <= 0 || gw <= 0) { dm::set_error("dm_beit_rel_table: bad arguments"); return DM_E_INVALID; }
    dm::beit_rel_table_host(table_host, window, heads, gh, gw, out_host);
    return DM_OK;
}
