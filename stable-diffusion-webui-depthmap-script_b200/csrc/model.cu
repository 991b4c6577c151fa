// §8(b) — the model-level C-ABI: dm_model_create / dm_depth_forward / dm_model_destroy.
//
// A dm_model owns everything a forward needs: the checkpoint packed into the kernels' layouts (fp16 GEMM operands,
// (ky,kx,cin)-ordered conv filters, ConvTranspose as GEMM + pixel shuffle, fp32 biases / LayerScale / tables), the
// activation buffers of the last (B, net) shape, the resolution-dependent tables (DINOv2 position embedding, BEiT
// relative-position tables) and one captured CUDA graph per (B, H, W, net, out) shape.  A forward is ONE C call:
// uint8 RGB images in device memory -> float32 prediction in device memory, asynchronous on the caller's stream.
//   replaces  ModelHolder.get_raw_prediction's network part (src/depthmap_generation.py:375-403) for
//     model types 12 / 13 / 14  estimatedepthanything_v2 (:548-559) + DepthAnythingV2.image2tensor / forward
//                               (ddepth_anything_v2/depth_anything_v2/dpt.py:117-221, dinov2.py:179-321)
//     model types 1 / 2         estimatemidas (:455-499) + DPTDepthModel.forward (dmidas/dpt_depth.py:110-166,
//                               dmidas/backbones/beit.py:18-129, dmidas/backbones/utils.py:28-249)
// The launch sequence is the one of the Python engines (depthmap_generation.py: run_network / run_head), which stay as
// the building-block path (ZoeDepth composes them) and as the A/B reference of tests/test_model_cabi_gpu.py.
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"

namespace dm {

static int ru(int x, int m) { return (x + m - 1) / m * m; }

struct ModelCfg {
    int family;            // 0 = Depth-Anything-V2 (DINOv2 + DPT head), 1 = MiDaS 3.1 DPT-BEiT, 2 = MiDaS 3.0 DPT-ViT (dpt_large_384)
    int C, depth, heads, Fch, oc[4], layers[4], window, patch;
    float mean[3], stdv[3];
    int final_mode;        // dm_resize_f32 mode
    const char *name;
};

static bool model_cfg(int model_type, ModelCfg &c) {
    const float im_mean[3] = {0.485f, 0.456f, 0.406f}, im_std[3] = {0.229f, 0.224f, 0.225f}, half3[3] = {0.5f, 0.5f, 0.5f};
    auto set = [&](int family, int C, int depth, int heads, int Fch, std::initializer_list<int> oc, std::initializer_list<int> layers, int window,
                   int patch, const float *m, const float *s, int final_mode, const char *name) {
        c.family = family; c.C = C; c.depth = depth; c.heads = heads; c.Fch = Fch; c.window = window; c.patch = patch; c.final_mode = final_mode; c.name = name;
        int i = 0; for (int v : oc) c.oc[i++] = v;
        i = 0; for (int v : layers) c.layers[i++] = v;
        for (int k = 0; k < 3; ++k) { c.mean[k] = m[k]; c.stdv[k] = s[k]; }
    };
    switch (model_type) {
        case 12: set(0, 384, 12, 6, 64, {48, 96, 192, 384}, {2, 5, 8, 11}, 0, 14, im_mean, im_std, 0, "depth_anything_v2_vits"); return true;
        case 13: set(0, 768, 12, 12, 128, {96, 192, 384, 768}, {2, 5, 8, 11}, 0, 14, im_mean, im_std, 0, "depth_anything_v2_vitb"); return true;
        case 14: set(0, 1024, 24, 16, 256, {256, 512, 1024, 1024}, {4, 11, 17, 23}, 0, 14, im_mean, im_std, 0, "depth_anything_v2_vitl"); return true;
        case 1: set(1, 1024, 24, 16, 256, {256, 512, 1024, 1024}, {5, 11, 17, 23}, 32, 16, half3, half3, 1, "dpt_beit_large_512"); return true;
        case 2: set(1, 1024, 24, 16, 256, {256, 512, 1024, 1024}, {5, 11, 17, 23}, 24, 16, half3, half3, 1, "dpt_beit_large_384"); return true;
        case 3: set(2, 1024, 24, 16, 256, {256, 512, 1024, 1024}, {5, 11, 17, 23}, 24, 16, half3, half3, 1, "dpt_large_384"); return true;
        case -100: set(1, 128, 4, 2, 64, {64, 64, 128, 128}, {0, 1, 2, 3}, 4, 16, half3, half3, 1, "beit_tiny (structural test configuration)"); return true;
        case -101: set(2, 128, 4, 2, 64, {64, 64, 128, 128}, {0, 1, 2, 3}, 4, 16, half3, half3, 1, "vit_tiny (structural test configuration)"); return true;
    }
    return false;
}

struct Weights {
    const dm_weight_blob *blob;
    std::map<std::string, const dm_weight *> idx;
    explicit Weights(const dm_weight_blob *b) : blob(b) { for (int i = 0; i < b->count; ++i) idx[b->items[i].name] = &b->items[i]; }
    const dm_weight *find(const std::string &k) const { auto it = idx.find(k); return it == idx.end() ? nullptr : it->second; }
    static int64_t numel(const dm_weight *w) { int64_t n = 1; for (int i = 0; i < w->ndim; ++i) n *= w->shape[i]; return n; }
    // element i of a tensor as float (dtype 0 = fp32, 1 = fp16, 2 = bf16)
    static float at(const dm_weight *w, int64_t i) {
        if (w->dtype == 0) return ((const float *)w->data_host)[i];
        if (w->dtype == 1) return __half2float(((const __half *)w->data_host)[i]);
        uint32_t u = (uint32_t)((const uint16_t *)w->data_host)[i] << 16;
        float f; memcpy(&f, &u, 4); return f;
    }
};

struct Block {
    float *ln1_w, *ln1_b, *qkv_b, *proj_b, *ls1, *ln2_w, *ln2_b, *fc1_b, *fc2_b, *ls2;
    __half *qkv_w, *proj_w, *fc1_w, *fc2_w;
    std::vector<float> rel_table_host;   // BEiT: [nrd, heads] as in the checkpoint
};

struct Buffers {
    int B = 0, nh = 0, nw = 0;
    std::map<std::string, void *> m;
    int sizes[4][2], up[4][2];
};

struct GraphKey { int B, H, W, nw, nh, oh, ow; bool operator<(const GraphKey &o) const { return std::tie(B, H, W, nw, nh, oh, ow) < std::tie(o.B, o.H, o.W, o.nw, o.nh, o.oh, o.ow); } };
struct GraphEntry { cudaGraphExec_t exec = nullptr; void *in = nullptr; float *out = nullptr; int calls = 0; };

}  // namespace dm

struct dm_model {
    dm::ModelCfg cfg;
    int model_type, device;
    std::vector<void *> owned;                 // weights + tables
    std::vector<void *> buf_owned;             // activation buffers of the current shape
    std::vector<dm::Block> blocks;
    std::map<std::string, void *> w;           // packed tensors by role
    std::vector<float> pos_embed_host;         // DINOv2 [1 + n*n, C]
    int pos_n = 0;
    float oc3_b = 0.f;
    int kpad = 0, ocp[4], Fp = 0, F2p = 0;
    dm::Buffers bufs;
    // resolution-dependent tables
    int tab_gh = -1, tab_gw = -1, nrd = 0;
    std::vector<float *> rel_tab;              // per block, device [heads, nrd] * log2e
    std::vector<void *> tab_owned;             // tables of the current resolution
    float *pos_dev = nullptr; int pos_gh = -1, pos_gw = -1;
    std::map<dm::GraphKey, dm::GraphEntry> graphs;
    cudaStream_t cap_stream = nullptr;         // graphs are captured on the model's own stream (the caller's may be the legacy default stream, which cannot capture)
    long long launches = 0;
};

namespace dm {

// ---- allocation / upload helpers -------------------------------------------------------------------------------
static int dev_alloc(std::vector<void *> &own, size_t bytes, void **out) {
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc (model)");
    own.push_back(p);
    *out = p;
    return DM_OK;
}
static int upload(std::vector<void *> &own, const void *host, size_t bytes, void **out) {
    int rc = dev_alloc(own, bytes, out);
    if (rc) return rc;
    cudaError_t e = cudaMemcpy(*out, host, bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpy (model weights)");
    return DM_OK;
}
#define DM_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// [rows, cols] matrix (row-major view of the checkpoint tensor) -> fp16 [rpad, cpad], zero padded
static int pack_mat(dm_model *m, const Weights &W, const std::string &key, int rows, int cols, int rpad, int cpad, __half **out) {
    const dm_weight *w = W.find(key);
    if (!w || Weights::numel(w) != (int64_t)rows * cols) { set_error("dm_model_create: weight '%s' missing or of unexpected size", key.c_str()); return DM_E_INVALID; }
    std::vector<__half> h((size_t)rpad * cpad, __float2half_rn(0.f));
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) h[(size_t)r * cpad + c] = __float2half_rn(Weights::at(w, (int64_t)r * cols + c));
    return upload(m->owned, h.data(), h.size() * sizeof(__half), (void **)out);
}
static int pack_vec(dm_model *m, const Weights &W, const std::string &key, int n, int npad, float **out, int repeat = 1) {
    const dm_weight *w = W.find(key);
    if (!w || Weights::numel(w) != n) { set_error("dm_model_create: weight '%s' missing or of unexpected size", key.c_str()); return DM_E_INVALID; }
    std::vector<float> v((size_t)npad * repeat, 0.f);
    for (int r = 0; r < repeat; ++r)
        for (int i = 0; i < n; ++i) v[(size_t)r * npad + i] = Weights::at(w, i);
    return upload(m->owned, v.data(), v.size() * sizeof(float), (void **)out);
}
static int const_vec(dm_model *m, float value, int n, float **out) {
    std::vector<float> v((size_t)n, value);
    return upload(m->owned, v.data(), v.size() * sizeof(float), (void **)out);
}
// conv filter [Cout, Cin, 3, 3] -> fp16 [cout_pad, 9 * cin_pad], K ordered (ky, kx, cin)
static int pack_conv3(dm_model *m, const Weights &W, const std::string &key, int co, int ci, int cop, int cip, __half **out) {
    const dm_weight *w = W.find(key);
    if (!w || Weights::numel(w) != (int64_t)co * ci * 9) { set_error("dm_model_create: weight '%s' missing or of unexpected size", key.c_str()); return DM_E_INVALID; }
    std::vector<__half> h((size_t)cop * 9 * cip, __float2half_rn(0.f));
    for (int o = 0; o < co; ++o)
        for (int i = 0; i < ci; ++i)
            for (int t = 0; t < 9; ++t) h[((size_t)o * 9 + t) * cip + i] = __float2half_rn(Weights::at(w, ((int64_t)o * ci + i) * 9 + t));
    return upload(m->owned, h.data(), h.size() * sizeof(__half), (void **)out);
}
// ConvTranspose2d(k = s) weight [Cin, Cout, s, s] -> fp16 [(i, j, co_pad), ci_pad]
static int pack_convT(dm_model *m, const Weights &W, const std::string &key, int c, int cp, int s, __half **out) {
    const dm_weight *w = W.find(key);
    if (!w || Weights::numel(w) != (int64_t)c * c * s * s) { set_error("dm_model_create: weight '%s' missing or of unexpected size", key.c_str()); return DM_E_INVALID; }
    std::vector<__half> h((size_t)s * s * cp * cp, __float2half_rn(0.f));
    for (int ci = 0; ci < c; ++ci)
        for (int co = 0; co < c; ++co)
            for (int i = 0; i < s; ++i)
                for (int j = 0; j < s; ++j)
                    h[(((size_t)i * s + j) * cp + co) * cp + ci] = __float2half_rn(Weights::at(w, (((int64_t)ci * c + co) * s + i) * s + j));
    return upload(m->owned, h.data(), h.size() * sizeof(__half), (void **)out);
}

// ---- checkpoint -> packed weights ---------------------------------------------------------------------------------
static int pack_model(dm_model *m, const Weights &W) {
    const ModelCfg &c = m->cfg;
    const int C = c.C, Fch = c.Fch;
    const bool beit = c.family == 1, vit = c.family == 2, midas = beit || vit;
    const std::string tp = midas ? "pretrained.model." : "pretrained.";
    const int kraw = 3 * c.patch * c.patch;
    m->kpad = ru(kraw, 64);
    __half *h; float *f;
    DM_TRY(pack_mat(m, W, tp + "patch_embed.proj.weight", C, kraw, C, m->kpad, &h)); m->w["pe_w"] = h;
    DM_TRY(pack_vec(m, W, tp + "patch_embed.proj.bias", C, C, &f)); m->w["pe_b"] = f;
    DM_TRY(pack_vec(m, W, tp + "cls_token", C, C, &f)); m->w["cls"] = f;
    if (!beit) {
        const dm_weight *pe = W.find(tp + "pos_embed");
        if (!pe || pe->ndim < 2) { set_error("dm_model_create: pretrained.pos_embed missing"); return DM_E_INVALID; }
        const int64_t n = Weights::numel(pe);
        const int tokens = (int)(n / C);
        m->pos_n = (int)llround(sqrt((double)(tokens - 1)));
        if ((int64_t)tokens * C != n || m->pos_n * m->pos_n != tokens - 1) { set_error("dm_model_create: pos_embed has an unexpected shape"); return DM_E_INVALID; }
        m->pos_embed_host.resize((size_t)n);
        for (int64_t i = 0; i < n; ++i) m->pos_embed_host[(size_t)i] = Weights::at(pe, i);
    }
    m->blocks.resize(c.depth);
    for (int i = 0; i < c.depth; ++i) {
        Block &b = m->blocks[i];
        const std::string p = tp + "blocks." + std::to_string(i) + ".";
        DM_TRY(pack_vec(m, W, p + "norm1.weight", C, C, &b.ln1_w)); DM_TRY(pack_vec(m, W, p + "norm1.bias", C, C, &b.ln1_b));
        DM_TRY(pack_vec(m, W, p + "norm2.weight", C, C, &b.ln2_w)); DM_TRY(pack_vec(m, W, p + "norm2.bias", C, C, &b.ln2_b));
        DM_TRY(pack_mat(m, W, p + "attn.qkv.weight", 3 * C, C, 3 * C, C, &b.qkv_w));
        DM_TRY(pack_mat(m, W, p + "attn.proj.weight", C, C, C, C, &b.proj_w)); DM_TRY(pack_vec(m, W, p + "attn.proj.bias", C, C, &b.proj_b));
        DM_TRY(pack_mat(m, W, p + "mlp.fc1.weight", 4 * C, C, 4 * C, C, &b.fc1_w)); DM_TRY(pack_vec(m, W, p + "mlp.fc1.bias", 4 * C, 4 * C, &b.fc1_b));
        DM_TRY(pack_mat(m, W, p + "mlp.fc2.weight", C, 4 * C, C, 4 * C, &b.fc2_w)); DM_TRY(pack_vec(m, W, p + "mlp.fc2.bias", C, C, &b.fc2_b));
        if (beit) {
            // qkv bias = cat(q_bias, zeros, v_bias): the key projection has no bias (dmidas/backbones/beit.py:70-74)
            const dm_weight *qb = W.find(p + "attn.q_bias"), *vb = W.find(p + "attn.v_bias");
            if (!qb || !vb) { set_error("dm_model_create: %sattn.q_bias / v_bias missing", p.c_str()); return DM_E_INVALID; }
            std::vector<float> v((size_t)3 * C, 0.f);
            for (int k = 0; k < C; ++k) { v[k] = Weights::at(qb, k); v[2 * C + k] = Weights::at(vb, k); }
            DM_TRY(upload(m->owned, v.data(), v.size() * 4, (void **)&b.qkv_b));
            DM_TRY(pack_vec(m, W, p + "gamma_1", C, C, &b.ls1)); DM_TRY(pack_vec(m, W, p + "gamma_2", C, C, &b.ls2));
            const dm_weight *rt = W.find(p + "attn.relative_position_bias_table");
            const int nrd0 = (2 * c.window - 1) * (2 * c.window - 1) + 3;
            if (!rt || Weights::numel(rt) != (int64_t)nrd0 * c.heads) { set_error("dm_model_create: %sattn.relative_position_bias_table missing or of unexpected size", p.c_str()); return DM_E_INVALID; }
            b.rel_table_host.resize((size_t)nrd0 * c.heads);
            for (size_t k = 0; k < b.rel_table_host.size(); ++k) b.rel_table_host[k] = Weights::at(rt, (int64_t)k);
        } else if (vit) {      // timm VisionTransformer block: full qkv bias, no LayerScale
            DM_TRY(pack_vec(m, W, p + "attn.qkv.bias", 3 * C, 3 * C, &b.qkv_b));
            DM_TRY(const_vec(m, 1.f, C, &b.ls1)); DM_TRY(const_vec(m, 1.f, C, &b.ls2));
        } else {
            DM_TRY(pack_vec(m, W, p + "attn.qkv.bias", 3 * C, 3 * C, &b.qkv_b));
            DM_TRY(pack_vec(m, W, p + "ls1.gamma", C, C, &b.ls1)); DM_TRY(pack_vec(m, W, p + "ls2.gamma", C, C, &b.ls2));
        }
    }
    if (midas) { DM_TRY(const_vec(m, 1.f, C, &f)); m->w["norm_w"] = f; DM_TRY(const_vec(m, 0.f, C, &f)); m->w["norm_b"] = f; }   // hooks read raw block outputs
    else { DM_TRY(pack_vec(m, W, "pretrained.norm.weight", C, C, &f)); m->w["norm_w"] = f; DM_TRY(pack_vec(m, W, "pretrained.norm.bias", C, C, &f)); m->w["norm_b"] = f; }
    // ---- reassemble + DPT decoder; channel counts padded to multiples of 64 with zero weights ----
    for (int i = 0; i < 4; ++i) m->ocp[i] = ru(c.oc[i], 64);
    m->Fp = ru(Fch, 64); m->F2p = ru(Fch / 2, 64);
    auto key_proj = [&](int i, const char *wb) { return midas ? "pretrained.act_postprocess" + std::to_string(i + 1) + ".3." + wb : "depth_head.projects." + std::to_string(i) + "." + wb; };
    auto key_resize = [&](int i, const char *wb) { return midas ? "pretrained.act_postprocess" + std::to_string(i + 1) + ".4." + wb : "depth_head.resize_layers." + std::to_string(i) + "." + wb; };
    const std::string sc = midas ? "scratch." : "depth_head.scratch.";
    for (int i = 0; i < 4; ++i) {
        DM_TRY(pack_mat(m, W, key_proj(i, "weight"), c.oc[i], C, m->ocp[i], C, &h)); m->w["proj" + std::to_string(i) + "_w"] = h;
        DM_TRY(pack_vec(m, W, key_proj(i, "bias"), c.oc[i], m->ocp[i], &f)); m->w["proj" + std::to_string(i) + "_b"] = f;
    }
    const int ups[2] = {4, 2};
    for (int i = 0; i < 2; ++i) {
        DM_TRY(pack_convT(m, W, key_resize(i, "weight"), c.oc[i], m->ocp[i], ups[i], &h)); m->w["up" + std::to_string(i) + "_w"] = h;
        DM_TRY(pack_vec(m, W, key_resize(i, "bias"), c.oc[i], m->ocp[i], &f, ups[i] * ups[i])); m->w["up" + std::to_string(i) + "_b"] = f;
    }
    DM_TRY(pack_conv3(m, W, key_resize(3, "weight"), c.oc[3], c.oc[3], m->ocp[3], m->ocp[3], &h)); m->w["down3_w"] = h;
    DM_TRY(pack_vec(m, W, key_resize(3, "bias"), c.oc[3], m->ocp[3], &f)); m->w["down3_b"] = f;
    for (int i = 0; i < 4; ++i) { DM_TRY(pack_conv3(m, W, sc + "layer" + std::to_string(i + 1) + "_rn.weight", Fch, c.oc[i], m->Fp, m->ocp[i], &h)); m->w["rn" + std::to_string(i) + "_w"] = h; }
    for (int i = 1; i <= 4; ++i) {
        const std::string r = sc + "refinenet" + std::to_string(i) + ".", rk = "rf" + std::to_string(i);
        DM_TRY(pack_mat(m, W, r + "out_conv.weight", Fch, Fch, m->Fp, m->Fp, &h)); m->w[rk + "_out_w"] = h;
        DM_TRY(pack_vec(m, W, r + "out_conv.bias", Fch, m->Fp, &f)); m->w[rk + "_out_b"] = f;
        for (int u = 1; u <= 2; ++u)
            for (int cv = 1; cv <= 2; ++cv) {
                const std::string k = r + "resConfUnit" + std::to_string(u) + ".conv" + std::to_string(cv) + ".";
                if (!W.find(k + "weight")) continue;        // refinenet4 has no resConfUnit1 in some exports
                const std::string rk2 = rk + "_u" + std::to_string(u) + "c" + std::to_string(cv);
                DM_TRY(pack_conv3(m, W, k + "weight", Fch, Fch, m->Fp, m->Fp, &h)); m->w[rk2 + "_w"] = h;
                DM_TRY(pack_vec(m, W, k + "bias", Fch, m->Fp, &f)); m->w[rk2 + "_b"] = f;
            }
    }
    const std::string oc1 = midas ? "scratch.output_conv.0." : "depth_head.scratch.output_conv1.";
    const std::string oc2 = midas ? "scratch.output_conv.2." : "depth_head.scratch.output_conv2.0.";
    const std::string oc3 = midas ? "scratch.output_conv.4." : "depth_head.scratch.output_conv2.2.";
    DM_TRY(pack_conv3(m, W, oc1 + "weight", Fch / 2, Fch, m->F2p, m->Fp, &h)); m->w["oc1_w"] = h;
    DM_TRY(pack_vec(m, W, oc1 + "bias", Fch / 2, m->F2p, &f)); m->w["oc1_b"] = f;
    DM_TRY(pack_conv3(m, W, oc2 + "weight", 32, Fch / 2, 32, m->F2p, &h)); m->w["oc2_w"] = h;
    DM_TRY(pack_vec(m, W, oc2 + "bias", 32, 32, &f)); m->w["oc2_b"] = f;
    DM_TRY(pack_vec(m, W, oc3 + "weight", 32, 32, &f)); m->w["oc3_w"] = f;
    const dm_weight *b3 = W.find(oc3 + "bias");
    if (!b3) { set_error("dm_model_create: %sbias missing", oc3.c_str()); return DM_E_INVALID; }
    m->oc3_b = Weights::at(b3, 0);
    if (midas)
        for (int j = 0; j < 4; ++j) {
            const std::string a = "pretrained.act_postprocess" + std::to_string(j + 1) + ".0.project.0.";
            DM_TRY(pack_mat(m, W, a + "weight", C, 2 * C, C, 2 * C, &h)); m->w["ro" + std::to_string(j) + "_w"] = h;
            DM_TRY(pack_vec(m, W, a + "bias", C, C, &f)); m->w["ro" + std::to_string(j) + "_b"] = f;
        }
    return DM_OK;
}

// ---- sizes (dmidas/transforms.py:61-104, util/transform.py:61-104) ---------------------------------------------------
static int constrain(double x, int mult, int min_val) {
    int y = (int)(nearbyint(x / mult) * mult);          // np.round: half to even
    if (y < min_val) y = (int)(ceil(x / mult) * mult);
    return y;
}
static void net_size(const ModelCfg &c, int W, int H, int net_w, int net_h, int *nw, int *nh) {
    if (c.family == 0) {       // Resize(lower_bound, multiple of 14); estimatedepthanything_v2 passes w as input_size (:552)
        double sh = (double)net_w / H, sw = (double)net_w / W;
        if (sw > sh) sh = sw; else sw = sh;
        *nw = constrain(sw * W, 14, net_w); *nh = constrain(sh * H, 14, net_w);
    } else {                   // Resize(minimal, multiple of 32)
        double sh = (double)net_h / H, sw = (double)net_w / W;
        if (fabs(1 - sw) < fabs(1 - sh)) sh = sw; else sw = sh;
        *nw = constrain(sw * W, 32, 0); *nh = constrain(sh * H, 32, 0);
    }
}

// ---- resolution-dependent tables ----------------------------------------------------------------------------------------
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

static int ensure_rel_tables(dm_model *m, int gh, int gw) {
    if (m->tab_gh == gh && m->tab_gw == gw) return DM_OK;
    const ModelCfg &c = m->cfg;
    const int nrd = (2 * gh - 1) * (2 * gw - 1) + 3, heads = c.heads;
    m->rel_tab.assign(c.depth, nullptr);
    for (void *p : m->tab_owned) cudaFree(p);      // the tables of the previous resolution (no graph of that resolution survives: ensure_buffers ran first)
    m->tab_owned.clear();
    std::vector<float> out((size_t)heads * nrd);
    for (int i = 0; i < c.depth; ++i) {
        beit_rel_table_host(m->blocks[i].rel_table_host.data(), c.window, heads, gh, gw, out.data());
        DM_TRY(upload(m->tab_owned, out.data(), out.size() * 4, (void **)&m->rel_tab[i]));
    }
    m->tab_gh = gh; m->tab_gw = gw; m->nrd = nrd;
    return DM_OK;
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

static int ensure_pos(dm_model *m, int gh, int gw) {
    if (m->pos_gh == gh && m->pos_gw == gw) return DM_OK;
    const int C = m->cfg.C;
    std::vector<float> out((size_t)(gh * gw + 1) * C);
    if (m->cfg.family == 2) vit_pos_embed_host(m->pos_embed_host.data(), m->pos_n, C, gh, gw, out.data());
    else dinov2_pos_embed_host(m->pos_embed_host.data(), m->pos_n, C, gh, gw, out.data());
    for (void *p : m->tab_owned) cudaFree(p);
    m->tab_owned.clear();
    DM_TRY(upload(m->tab_owned, out.data(), out.size() * 4, (void **)&m->pos_dev));
    m->pos_gh = gh; m->pos_gw = gw;
    return DM_OK;
}

// ---- activation buffers ----------------------------------------------------------------------------------------------------
static int ensure_buffers(dm_model *m, int B, int nh, int nw) {
    Buffers &b = m->bufs;
    if (b.B == B && b.nh == nh && b.nw == nw) return DM_OK;
    for (void *p : m->buf_owned) cudaFree(p);
    m->buf_owned.clear(); b.m.clear(); b.B = 0;
    for (auto &g : m->graphs) if (g.second.exec) cudaGraphExecDestroy(g.second.exec);   // graphs point into the old buffers
    m->graphs.clear();
    const ModelCfg &c = m->cfg;
    const int C = c.C, Fp = m->Fp, gh = nh / c.patch, gw = nw / c.patch, Np = gh * gw, N = Np + 1;
    auto A = [&](const std::string &k, size_t bytes) { void *p; int rc = dev_alloc(m->buf_owned, bytes, &p); if (!rc) b.m[k] = p; return rc; };
    const size_t h = sizeof(__half);
    DM_TRY(A("patches", (size_t)B * Np * m->kpad * h)); DM_TRY(A("pe", (size_t)B * Np * C * h)); DM_TRY(A("x", (size_t)B * N * C * 4));
    DM_TRY(A("h", (size_t)B * N * C * h)); DM_TRY(A("qkv", (size_t)B * N * 3 * C * h)); DM_TRY(A("att", (size_t)B * N * C * h));
    DM_TRY(A("mlp", (size_t)B * N * 4 * C * h));
    for (int i = 0; i < 4; ++i) DM_TRY(A("feat" + std::to_string(i), (size_t)B * Np * C * h));
    if (c.family != 0) DM_TRY(A("cat", (size_t)B * Np * 2 * C * h));
    const int sz[4][2] = {{gh * 4, gw * 4}, {gh * 2, gw * 2}, {gh, gw}, {(gh - 1) / 2 + 1, (gw - 1) / 2 + 1}};
    memcpy(b.sizes, sz, sizeof(sz));
    const int up[4][2] = {{sz[2][0], sz[2][1]}, {sz[1][0], sz[1][1]}, {sz[0][0], sz[0][1]}, {sz[0][0] * 2, sz[0][1] * 2}};
    memcpy(b.up, up, sizeof(up));
    for (int i = 0; i < 4; ++i) DM_TRY(A("p" + std::to_string(i), (size_t)B * Np * m->ocp[i] * h));
    DM_TRY(A("r0", (size_t)B * sz[0][0] * sz[0][1] * m->ocp[0] * h)); DM_TRY(A("r1", (size_t)B * sz[1][0] * sz[1][1] * m->ocp[1] * h));
    DM_TRY(A("r3", (size_t)B * sz[3][0] * sz[3][1] * m->ocp[3] * h)); DM_TRY(A("cols3", (size_t)B * sz[3][0] * sz[3][1] * 9 * m->ocp[3] * h));
    for (int i = 0; i < 4; ++i) {
        const size_t px = (size_t)B * sz[i][0] * sz[i][1] * Fp * h;
        const std::string s = std::to_string(i);
        DM_TRY(A("l" + s, px)); DM_TRY(A("lr" + s, px)); DM_TRY(A("t" + s, px)); DM_TRY(A("o" + s, px)); DM_TRY(A("or" + s, px)); DM_TRY(A("u" + s, px));
    }
    const int vs[4] = {3, 2, 1, 0};
    for (int i = 0; i < 4; ++i) {
        DM_TRY(A("v" + std::to_string(i), (size_t)B * sz[vs[i]][0] * sz[vs[i]][1] * Fp * h));
        DM_TRY(A("path" + std::to_string(i), (size_t)B * up[i][0] * up[i][1] * Fp * h));
    }
    DM_TRY(A("oc1", (size_t)B * up[3][0] * up[3][1] * m->F2p * h)); DM_TRY(A("oc1u", (size_t)B * nh * nw * m->F2p * h));
    DM_TRY(A("d", (size_t)B * nh * nw * 4));
    b.B = B; b.nh = nh; b.nw = nw;
    return DM_OK;
}

// ---- the launch sequence (mirrors DepthAnythingV2Engine.run_network / run_head) --------------------------------------------
static int gemm(dm_model *m, const void *A, int lda, const void *Wt, int ldw, int M, int N, int K, cudaStream_t s, int epi = DM_EPI_STORE_F16,
                int act = DM_ACT_NONE, const float *bias = nullptr, void *C = nullptr, int ldc = 0, float *X = nullptr, int ldx = 0, const float *gamma = nullptr,
                int ps_s = 0, int ps_c = 0, int ps_h = 0, int ps_w = 0) {
    dm_gemm_desc d;
    memset(&d, 0, sizeof(d));
    d.M = M; d.N = N; d.K = K; d.epi = epi; d.act = act; d.bias = bias; d.C = C; d.ldc = ldc; d.X = X; d.ldx = ldx; d.gamma = gamma;
    d.ps_s = ps_s; d.ps_cout = ps_c; d.ps_h = ps_h; d.ps_w = ps_w;
    ++m->launches;
    return dm_gemm_ex(A, lda, Wt, ldw, &d, s);
}
static int conv(dm_model *m, const void *act_t, int B, int H, int W, int Cin, const void *Wt, int Cout, cudaStream_t s, int epi = DM_EPI_STORE_F16,
                int act = DM_ACT_NONE, const float *bias = nullptr, void *C = nullptr, void *C2 = nullptr, const void *R = nullptr, const void *R2 = nullptr,
                float *X = nullptr, const float *gamma = nullptr, float head_b2 = 0.f) {
    dm_gemm_desc d;
    memset(&d, 0, sizeof(d));
    d.N = Cout; d.epi = epi; d.act = act; d.bias = bias; d.C = C; d.ldc = Cout; d.C2 = C2; d.R = R; d.ldr = Cout; d.R2 = R2; d.ldr2 = Cout;
    d.X = X; d.ldx = 1; d.gamma = gamma; d.head_b2 = head_b2;
    ++m->launches;
    return dm_conv3x3_ex(act_t, B, H, W, Cin, Wt, &d, s);
}

static int run_forward(dm_model *m, const uint8_t *rgb, int B, int H, int W, int nw, int nh, float *out, int oh, int ow, cudaStream_t st) {
    const ModelCfg &c = m->cfg;
    Buffers &b = m->bufs;
    auto W_ = [&](const std::string &k) { return m->w.at(k); };
    auto Bf = [&](const std::string &k) { return b.m.at(k); };
    const int C = c.C, heads = c.heads, Fp = m->Fp, P = c.patch, gh = nh / P, gw = nw / P, Np = gh * gw, N = Np + 1;
    const bool beit = c.family == 1, midas = c.family != 0;
    const int cmap[3] = {2, 1, 0};   // the reference swaps R/B an odd number of times before the network sees the image (:381,550; dpt.py:213)
    DM_TRY(dm_preprocess_patchify(rgb, B, H, W, nh, nw, P, c.mean, c.stdv, cmap, Bf("patches"), m->kpad, st));
    m->launches += m->kpad > 3 * P * P ? 2 : 1;
    DM_TRY(gemm(m, Bf("patches"), m->kpad, W_("pe_w"), m->kpad, B * Np, C, m->kpad, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_("pe_b"), Bf("pe"), C));
    DM_TRY(dm_assemble_tokens(Bf("pe"), (float *)W_("cls"), beit ? nullptr : m->pos_dev, (float *)Bf("x"), B, Np, C, st));
    ++m->launches;
    const long long rows = (long long)B * N;
    const float scale = 1.0f / sqrtf((float)(C / heads));
    int fi = 0;
    for (int i = 0; i < c.depth; ++i) {
        const Block &k = m->blocks[i];
        DM_TRY(dm_layernorm_f16((float *)Bf("x"), rows, C, k.ln1_w, k.ln1_b, 1e-6f, Bf("h"), 1, 0, st));
        DM_TRY(gemm(m, Bf("h"), C, k.qkv_w, C, (int)rows, 3 * C, C, st, DM_EPI_STORE_F16, DM_ACT_NONE, k.qkv_b, Bf("qkv"), 3 * C));
        if (beit) DM_TRY(dm_attention_relpos_f16(Bf("qkv"), B, gh, gw, heads, scale, m->rel_tab[i], m->nrd, Bf("att"), st));
        else DM_TRY(dm_attention_f16(Bf("qkv"), B, N, heads, scale, nullptr, 0, Bf("att"), st));
        DM_TRY(gemm(m, Bf("att"), C, k.proj_w, C, (int)rows, C, C, st, DM_EPI_RESID_F32, DM_ACT_NONE, k.proj_b, nullptr, 0, (float *)Bf("x"), C, k.ls1));
        DM_TRY(dm_layernorm_f16((float *)Bf("x"), rows, C, k.ln2_w, k.ln2_b, 1e-6f, Bf("h"), 1, 0, st));
        DM_TRY(gemm(m, Bf("h"), C, k.fc1_w, C, (int)rows, 4 * C, C, st, DM_EPI_STORE_F16, DM_ACT_GELU, k.fc1_b, Bf("mlp"), 4 * C));
        DM_TRY(gemm(m, Bf("mlp"), 4 * C, k.fc2_w, 4 * C, (int)rows, C, 4 * C, st, DM_EPI_RESID_F32, DM_ACT_NONE, k.fc2_b, nullptr, 0, (float *)Bf("x"), C, k.ls2));
        m->launches += 3;
        if (fi < 4 && i == c.layers[fi]) {
            const std::string f = "feat" + std::to_string(fi);
            if (midas) {  // forward hook on the raw block output + ProjectReadout: GELU(Linear(cat(tokens, cls)))
                DM_TRY(dm_concat_readout_f16((float *)Bf("x"), B, N, C, Bf("cat"), st));
                DM_TRY(gemm(m, Bf("cat"), 2 * C, W_("ro" + std::to_string(fi) + "_w"), 2 * C, B * Np, C, 2 * C, st, DM_EPI_STORE_F16, DM_ACT_GELU,
                            (float *)W_("ro" + std::to_string(fi) + "_b"), Bf(f), C));
            } else {      // get_intermediate_layers(norm=True) without the class token
                DM_TRY(dm_layernorm_f16((float *)Bf("x"), rows, C, (float *)W_("norm_w"), (float *)W_("norm_b"), 1e-6f, Bf(f), N, 1, st));
            }
            ++m->launches;
            ++fi;
        }
    }
    // ---- reassemble ----
    const int (*sz)[2] = b.sizes;
    for (int i = 0; i < 4; ++i) {
        const std::string s = std::to_string(i);
        DM_TRY(gemm(m, Bf("feat" + s), C, W_("proj" + s + "_w"), C, B * Np, m->ocp[i], C, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_("proj" + s + "_b"), Bf("p" + s), m->ocp[i]));
    }
    DM_TRY(gemm(m, Bf("p0"), m->ocp[0], W_("up0_w"), m->ocp[0], B * Np, 16 * m->ocp[0], m->ocp[0], st, DM_EPI_PIXSHUF, DM_ACT_NONE, (float *)W_("up0_b"), Bf("r0"), 0,
                nullptr, 0, nullptr, 4, m->ocp[0], gh, gw));
    DM_TRY(gemm(m, Bf("p1"), m->ocp[1], W_("up1_w"), m->ocp[1], B * Np, 4 * m->ocp[1], m->ocp[1], st, DM_EPI_PIXSHUF, DM_ACT_NONE, (float *)W_("up1_b"), Bf("r1"), 0,
                nullptr, 0, nullptr, 2, m->ocp[1], gh, gw));
    DM_TRY(dm_im2col_s2_f16(Bf("p3"), B, gh, gw, m->ocp[3], Bf("cols3"), st));
    ++m->launches;
    DM_TRY(gemm(m, Bf("cols3"), 9 * m->ocp[3], W_("down3_w"), 9 * m->ocp[3], B * sz[3][0] * sz[3][1], m->ocp[3], 9 * m->ocp[3], st, DM_EPI_STORE_F16, DM_ACT_NONE,
                (float *)W_("down3_b"), Bf("r3"), m->ocp[3]));
    const void *rs[4] = {Bf("r0"), Bf("r1"), Bf("p2"), Bf("r3")};
    for (int i = 0; i < 4; ++i) {
        const std::string s = std::to_string(i);
        DM_TRY(conv(m, rs[i], B, sz[i][0], sz[i][1], m->ocp[i], W_("rn" + s + "_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, nullptr, Bf("l" + s), Bf("lr" + s)));
    }
    // ---- fusion blocks; out_conv (1x1) runs BEFORE the up-sample (it commutes with bilinear interpolation) ----
    const int (*up)[2] = b.up;
    DM_TRY(conv(m, Bf("lr3"), B, sz[3][0], sz[3][1], Fp, W_("rf4_u2c1_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_RELU, (float *)W_("rf4_u2c1_b"), Bf("t3")));
    DM_TRY(conv(m, Bf("t3"), B, sz[3][0], sz[3][1], Fp, W_("rf4_u2c2_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_("rf4_u2c2_b"), Bf("u3"), nullptr, Bf("l3")));
    DM_TRY(gemm(m, Bf("u3"), Fp, W_("rf4_out_w"), Fp, B * sz[3][0] * sz[3][1], Fp, Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_("rf4_out_b"), Bf("v0"), Fp));
    DM_TRY(dm_resize_bilinear_nhwc_f16(Bf("v0"), B, sz[3][0], sz[3][1], Fp, Bf("path0"), up[0][0], up[0][1], st));
    ++m->launches;
    const int lis[3] = {2, 1, 0}, rfs[3] = {3, 2, 1};
    for (int step = 0; step < 3; ++step) {
        const int li = lis[step];
        const std::string s = std::to_string(li), rk = "rf" + std::to_string(rfs[step]);
        const int h_ = sz[li][0], w_ = sz[li][1];
        DM_TRY(conv(m, Bf("lr" + s), B, h_, w_, Fp, W_(rk + "_u1c1_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_RELU, (float *)W_(rk + "_u1c1_b"), Bf("t" + s)));
        DM_TRY(conv(m, Bf("t" + s), B, h_, w_, Fp, W_(rk + "_u1c2_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_(rk + "_u1c2_b"), Bf("o" + s), Bf("or" + s), Bf("l" + s),
                    Bf("path" + std::to_string(step))));
        DM_TRY(conv(m, Bf("or" + s), B, h_, w_, Fp, W_(rk + "_u2c1_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_RELU, (float *)W_(rk + "_u2c1_b"), Bf("t" + s)));
        DM_TRY(conv(m, Bf("t" + s), B, h_, w_, Fp, W_(rk + "_u2c2_w"), Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_(rk + "_u2c2_b"), Bf("u" + s), nullptr, Bf("o" + s)));
        DM_TRY(gemm(m, Bf("u" + s), Fp, W_(rk + "_out_w"), Fp, B * h_ * w_, Fp, Fp, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_(rk + "_out_b"), Bf("v" + std::to_string(step + 1)), Fp));
        DM_TRY(dm_resize_bilinear_nhwc_f16(Bf("v" + std::to_string(step + 1)), B, h_, w_, Fp, Bf("path" + std::to_string(step + 1)), up[step + 1][0], up[step + 1][1], st));
        ++m->launches;
    }
    // ---- output_conv + final resize ----
    DM_TRY(conv(m, Bf("path3"), B, up[3][0], up[3][1], Fp, W_("oc1_w"), m->F2p, st, DM_EPI_STORE_F16, DM_ACT_NONE, (float *)W_("oc1_b"), Bf("oc1")));
    DM_TRY(dm_resize_bilinear_nhwc_f16(Bf("oc1"), B, up[3][0], up[3][1], m->F2p, Bf("oc1u"), nh, nw, st));
    DM_TRY(conv(m, Bf("oc1u"), B, nh, nw, m->F2p, W_("oc2_w"), 32, st, DM_EPI_HEAD, DM_ACT_RELU, (float *)W_("oc2_b"), nullptr, nullptr, nullptr, nullptr, (float *)Bf("d"),
                (float *)W_("oc3_w"), m->oc3_b));
    DM_TRY(dm_resize_f32((float *)Bf("d"), B, nh, nw, out, oh, ow, c.final_mode, st));
    m->launches += 2;
    return DM_OK;
}

}  // namespace dm

#define DM_EXPORT extern "C" __attribute__((visibility("default")))

DM_EXPORT int dm_model_create(dm_model_t **out, int model_type, const dm_weight_blob *weights, int device, int dtype) {
    using namespace dm;
    if (!out || !weights || !weights->items || weights->count <= 0) { set_error("dm_model_create: bad arguments"); return DM_E_INVALID; }
    *out = nullptr;
    ModelCfg cfg;
    if (!model_cfg(model_type, cfg)) { set_error("dm_model_create: model_type %d has no native model (1, 2 = DPT-BEiT-L 512 / 384; 3 = DPT-Large 384; 12, 13, 14 = Depth-Anything-V2 S / B / L)", model_type); return DM_E_UNSUPPORTED; }
    if (dtype != 0) { set_error("dm_model_create: only dtype 0 (fp16 operands, fp32 accumulation and residual stream) is implemented"); return DM_E_UNSUPPORTED; }
    DM_CUDA_CHECK(cudaSetDevice(device));
    dm_model *m = new dm_model();
    m->cfg = cfg; m->model_type = model_type; m->device = device;
    Weights W(weights);
    const int rc = pack_model(m, W);
    if (rc) { dm_model_destroy(m); return rc; }
    *out = m;
    return DM_OK;
}

DM_EXPORT int dm_model_destroy(dm_model_t *m) {
    if (!m) return DM_OK;
    for (auto &g : m->graphs) { if (g.second.exec) cudaGraphExecDestroy(g.second.exec); }
    if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
    for (void *p : m->buf_owned) cudaFree(p);
    for (void *p : m->tab_owned) cudaFree(p);
    for (void *p : m->owned) cudaFree(p);
    delete m;
    return DM_OK;
}

/* resolution-dependent tables as the model builds them (host arithmetic); exported so the op-level path uses the very same numbers */
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

DM_EXPORT int dm_model_net_size(const dm_model_t *m, int W, int H, int net_w, int net_h, int *nw, int *nh) {
    if (!m || !nw || !nh) { dm::set_error("dm_model_net_size: bad arguments"); return DM_E_INVALID; }
    dm::net_size(m->cfg, W, H, net_w, net_h, nw, nh);
    return DM_OK;
}

DM_EXPORT long long dm_model_launches(const dm_model_t *m) { return m ? m->launches : 0; }

DM_EXPORT int dm_depth_forward(dm_model_t *m, const uint8_t *rgb, int B, int H, int W, int net_w, int net_h, float *depth_out, int out_h, int out_w, void *stream_) {
    using namespace dm;
    if (!m || !rgb || !depth_out || B <= 0 || H <= 0 || W <= 0 || net_w <= 0 || net_h <= 0 || out_h <= 0 || out_w <= 0) { set_error("dm_depth_forward: bad arguments"); return DM_E_INVALID; }
    cudaStream_t st = (cudaStream_t)stream_;
    int nw, nh;
    net_size(m->cfg, W, H, net_w, net_h, &nw, &nh);
    if (nw <= 0 || nh <= 0 || nw % m->cfg.patch || nh % m->cfg.patch) { set_error("dm_depth_forward: net size %dx%d is not a multiple of the patch size", nw, nh); return DM_E_INVALID; }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    const bool outer_capture = cap != cudaStreamCaptureStatusNone;
    const bool same_shape = m->bufs.B == B && m->bufs.nh == nh && m->bufs.nw == nw;
    if (outer_capture && !same_shape) { set_error("dm_depth_forward: run this shape once before capturing it into a CUDA graph (buffers are allocated on first use)"); return DM_E_INVALID; }
    const int gh = nh / m->cfg.patch, gw = nw / m->cfg.patch;
    if (!outer_capture) {
        DM_TRY(ensure_buffers(m, B, nh, nw));
        if (m->cfg.family == 1) DM_TRY(ensure_rel_tables(m, gh, gw)); else DM_TRY(ensure_pos(m, gh, gw));
    } else if ((m->cfg.family == 1 && (m->tab_gh != gh || m->tab_gw != gw)) || (m->cfg.family != 1 && (m->pos_gh != gh || m->pos_gw != gw))) {
        set_error("dm_depth_forward: resolution tables missing while capturing"); return DM_E_INVALID;
    }
    static int use_graph = -1;
    if (use_graph < 0) { const char *e = getenv("DEPTHMAP_B200_MODEL_GRAPH"); use_graph = (e && e[0] == '0') ? 0 : 1; }
    if (outer_capture || !use_graph) return run_forward(m, rgb, B, H, W, nw, nh, depth_out, out_h, out_w, st);
    // own graph: call 1 of a shape runs eagerly (and validates), call 2 captures, later calls replay.  The graph reads
    // the images from / writes the prediction to model-owned staging buffers, so caller pointers may change per call.
    GraphKey key{B, H, W, nw, nh, out_h, out_w};
    GraphEntry &g = m->graphs[key];
    ++g.calls;
    if (g.calls == 1) return run_forward(m, rgb, B, H, W, nw, nh, depth_out, out_h, out_w, st);
    const size_t in_bytes = (size_t)B * H * W * 3, out_bytes = (size_t)B * out_h * out_w * sizeof(float);
    if (!g.exec) {
        DM_TRY(dev_alloc(m->buf_owned, in_bytes, &g.in));
        DM_TRY(dev_alloc(m->buf_owned, out_bytes, (void **)&g.out));
        cudaGraph_t graph = nullptr;
        if (!m->cap_stream) DM_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        DM_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        const int rc = run_forward(m, (const uint8_t *)g.in, B, H, W, nw, nh, g.out, out_h, out_w, m->cap_stream);
        cudaError_t e = cudaStreamEndCapture(m->cap_stream, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (e != cudaSuccess) return cuda_fail(e, "cudaStreamEndCapture (dm_depth_forward)");
        e = cudaGraphInstantiate(&g.exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) { g.exec = nullptr; return cuda_fail(e, "cudaGraphInstantiate (dm_depth_forward)"); }
    }
    DM_CUDA_CHECK(cudaMemcpyAsync(g.in, rgb, in_bytes, cudaMemcpyDeviceToDevice, st));
    DM_CUDA_CHECK(cudaGraphLaunch(g.exec, st));
    DM_CUDA_CHECK(cudaMemcpyAsync(depth_out, g.out, out_bytes, cudaMemcpyDeviceToDevice, st));
    return DM_OK;
}
