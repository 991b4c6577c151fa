// Fused multi-head attention forward for the ViT backbones (head_dim 64, N <= a few thousand tokens, no mask):
//   O = softmax(scale * Q K^T [+ rel_pos_bias]) V
// Replaces the materialised attention of the reference (dinov2_layers/attention.py:49-62; dmidas/backbones/beit.py:65-91,
// which writes a [B,16,N,N] tensor per block and rebuilds the relative-position bias every forward).
//
// One CTA per (128-query tile, head, image), three warpgroups:
//   warpgroup 0    TMA producer (one thread): the Q tile once, then K_j / V_j tiles (128 keys x 64) into a 2-stage ring,
//                  straight out of the packed qkv activation [B*N, 3C] (no head split / transpose pass)
//   warpgroups 1-2 consumers, 64 query rows each, everything in registers:
//                    S  = Q K_j^T   wgmma m64n128k16, both operands K-major in shared memory, fp32 S fragment
//                    online softmax on the fragment (a query row lives in the four lanes of a quad: two shuffles per
//                    reduction), exp2 with the scale and log2 e folded in, running (max, sum), O rescaled in registers
//                    O += P V_j     wgmma m64n64k16 with A = P packed to fp16 in registers (the S fragment IS the A
//                    fragment layout, tc_common.cuh) and B = V_j used MN-major, so neither P nor V^T ever touches memory
// While one warpgroup exponentiates, the other one's MMAs keep the tensor cores busy.
// Bias modes: 0 none (DINOv2) | 1 dense fp16 [H,N,ld] | 2 BEiT relative-position table [H, nrd] (pre-multiplied by log2 e),
// any window: the bias of (q, k) is table[base_q - koff_k] with base_q = (qy+gh-1)(2gw-1) + qx+gw-1 and koff_k = ky(2gw-1) + kx,
// so no [H,N,N] tensor is ever read (the reference materialises it per block per forward).  A 128-query x 128-key tile pair
// needs only the table rows dy = qy - ky it spans, (query rows spanned + key rows spanned - 1) x (2gw - 1) contiguous entries
// (995 floats at 100 x 100).  Warps 1-3 of the producer warpgroup copy that sub-window out of the L2-resident table, with the
// key offsets rebased onto it (32-bit), into the same 2-stage ring as K / V and arrive on the stage's full barrier.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dm {
using namespace tc;

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

int make_tmap_2d(CUtensorMap *tm, const void *ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols);

struct AttnParams {
    int B, N, H;            // images, tokens per image, heads
    int C;                  // H * 64
    float scale_log2e;      // softmax scale * log2(e)
    const __half *bias;     // optional [H, N, bias_ld] additive bias (natural-log domain)
    int bias_ld;
    __half *out;            // [B*N, C]
    const float *rel_table; // optional [H, nrd] * log2(e): BEiT relative-position table
    int nrd, gh, gw;
    int sub_stride;         // mode 2: floats per stage of the streamed sub-window (the last one holds the class-query entry)
};

constexpr int AT_BQ = 128, AT_BKV = 128, AT_D = 64, AT_STAGES = 2;
constexpr int AT_THREADS = 384;
constexpr int AT_Q_BYTES = AT_BQ * AT_D * 2;        // 16 KB
constexpr int AT_KV_BYTES = AT_BKV * AT_D * 2;      // 16 KB each for K and V
constexpr int AT_K_OFF = AT_Q_BYTES;
constexpr int AT_V_OFF = AT_K_OFF + AT_STAGES * AT_KV_BYTES;
constexpr int AT_BAR_OFF = AT_V_OFF + AT_STAGES * AT_KV_BYTES;
constexpr int AT_TAB_OFF = AT_BAR_OFF + 64;         // mode 2: table sub-windows + key offsets, per stage
constexpr int AT_SMEM_MAX = 227 * 1024;
constexpr int AT_STAGERS = 96;                      // mode 2: producer warps 1-3 stage the table sub-windows

// mode 2: largest sub-window of a tile pair (+1 for the class-query entry), rounded to 16 bytes.  128 consecutive patch
// tokens cover at most 127 / gw + 2 grid rows, so a pair spans at most 2 * that - 1 offsets dy.
static inline int relpos_sub_stride(int gh, int gw) {
    const int span = gh < (AT_BQ - 1) / gw + 2 ? gh : (AT_BQ - 1) / gw + 2;
    return ((2 * span - 1) * (2 * gw - 1) + 1 + 3) & ~3;
}

template <int BIAS_MODE>
__global__ void __launch_bounds__(AT_THREADS, 1) attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, AttnParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *sQ = smem_raw, *sK = smem_raw + AT_K_OFF, *sV = smem_raw + AT_V_OFF;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + AT_BAR_OFF);
    uint64_t *q_full = bars, *kv_full = bars + 1, *kv_empty = bars + 1 + AT_STAGES;
    float *s_tab = reinterpret_cast<float *>(smem_raw + AT_TAB_OFF);                 // mode 2: [stage][sub_stride]
    int *s_koff = reinterpret_cast<int *>(s_tab + AT_STAGES * p.sub_stride);         // mode 2: [stage][128] after the sub-windows

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ, h = blockIdx.y, b = blockIdx.z;
    const int num_kv = (p.N + AT_BKV - 1) / AT_BKV;
    const int row_base = b * p.N;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmQKV);
        mbar_init(q_full, 1);
        for (int s = 0; s < AT_STAGES; ++s) {
            mbar_init(&kv_full[s], BIAS_MODE == 2 ? 1 + AT_STAGERS : 1);      // mode 2: + the table stagers
            mbar_init(&kv_empty[s], 8);                                       // 8 consumer warps
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(q_full, AT_Q_BYTES);
            tma_load_2d(sQ, &tmQKV, q_full, h * AT_D, row_base + q0);
            for (int j = 0; j < num_kv; ++j) {
                const int s = j % AT_STAGES;
                mbar_wait(&kv_empty[s], ((j / AT_STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(&kv_full[s], 2 * AT_KV_BYTES);
                tma_load_2d(sK + s * AT_KV_BYTES, &tmQKV, &kv_full[s], p.C + h * AT_D, row_base + j * AT_BKV);
                tma_load_2d(sV + s * AT_KV_BYTES, &tmQKV, &kv_full[s], 2 * p.C + h * AT_D, row_base + j * AT_BKV);
            }
        } else if (BIAS_MODE == 2 && warp >= 1) {
            // Every query / key tile holds at least one patch token (N >= 2); class and padding positions take the offsets of the
            // nearest patch token of their tile, so every index the consumers form stays inside the sub-window (the values they
            // read there are replaced or masked).
            const int st = threadIdx.x - 32, rw = 2 * p.gw - 1;
            const float *tab = p.rel_table + (size_t)h * p.nrd;
            const int qy_min = (max(q0, 1) - 1) / p.gw, qy_max = (min(q0 + AT_BQ, p.N) - 2) / p.gw;
            for (int j = 0; j < num_kv; ++j) {
                const int s = j % AT_STAGES, kbase = j * AT_BKV;
                const int k_lo = max(kbase, 1), k_hi = min(kbase + AT_BKV, p.N) - 1;
                const int ky_min = (k_lo - 1) / p.gw, ky_max = (k_hi - 1) / p.gw;
                const int lo = (qy_min - ky_max + p.gh - 1) * rw;                 // first table entry of the pair
                const int cnt = (qy_max - qy_min + ky_max - ky_min + 1) * rw;
                float *sub = s_tab + s * p.sub_stride;
                int *kof = s_koff + s * AT_BKV;
                mbar_wait(&kv_empty[s], ((j / AT_STAGES) & 1) ^ 1);
                for (int i = st; i < cnt; i += AT_STAGERS) sub[i] = __ldg(tab + lo + i);
                if (st == 0) sub[p.sub_stride - 1] = __ldg(tab + p.nrd - 3);      // class query -> patch key
                for (int k = st; k < AT_BKV; k += AT_STAGERS) {
                    const int t = min(max(kbase + k, k_lo), k_hi) - 1;
                    kof[k] = (t / p.gw) * rw + (t % p.gw) + lo;
                }
                mbar_arrive(&kv_full[s]);
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile; this thread rows r and r + 8 =====
    const int wg = (warp >> 2) - 1, t = lane & 3;
    constexpr float LOG2E = 1.4426950408889634f;
    int qi[2];
    bool q_ok[2];
    const __half *brow[2] = {nullptr, nullptr};
    int rp_base[2] = {0, 0}, rp_mult[2] = {1, 1};
    float rp_k0[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        qi[r] = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
        q_ok[r] = qi[r] < p.N;
        const int qq = q_ok[r] ? qi[r] : 0;
        if (BIAS_MODE == 1) brow[r] = p.bias + ((size_t)h * p.N + qq) * p.bias_ld;
        if (BIAS_MODE == 2) {
            // class-token query: the constant class->patch entry; class-token key: see the k == 0 case below
            // (dmidas/backbones/beit.py:44-62 assembles exactly these three extra entries).  The key offsets are rebased onto
            // each tile pair's sub-window, so the query base stays the full-table one; the class->patch entry sits in the
            // sub-window's last slot.
            const float *tab = p.rel_table + (size_t)h * p.nrd;
            if (qq == 0) { rp_base[r] = p.sub_stride - 1; rp_mult[r] = 0; rp_k0[r] = __ldg(tab + p.nrd - 1); }
            else {
                const int tt = qq - 1, qy = tt / p.gw, qx = tt % p.gw;
                rp_base[r] = (qy + p.gh - 1) * (2 * p.gw - 1) + (qx + p.gw - 1);
                rp_k0[r] = __ldg(tab + p.nrd - 2);
            }
        }
    }
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint64_t qdesc = make_desc_kmajor_sw128(smem_u32(sQ) + wg * (64 * 128));

    mbar_wait(q_full, 0);
    for (int j = 0; j < num_kv; ++j) {
        const int s = j % AT_STAGES;
        const int kbase = j * AT_BKV;
        mbar_wait(&kv_full[s], (j / AT_STAGES) & 1);
        // ---- S = Q K_j^T ---------------------------------------------------------------------------------------------
        float sc[64];
        const float *sub = s_tab + s * p.sub_stride;          // mode 2: this tile pair's table rows and rebased key offsets
        const int *kof = s_koff + s * AT_BKV;
        const uint64_t kdesc = make_desc_kmajor_sw128(smem_u32(sK + s * AT_KV_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_ss<AT_BKV>(sc, qdesc + (uint64_t)(2 * k), kdesc + (uint64_t)(2 * k), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        // ---- u = s * scale + bias (log2 domain), keys past the image masked, row maximum ------------------------------
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int c = 0; c < AT_BKV / 8; ++c) {
            const int k0 = kbase + 8 * c + 2 * t;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float b0 = 0.f, b1 = 0.f;
                if (BIAS_MODE == 1) {
                    const float2 bf = __half22float2(__ldg(reinterpret_cast<const __half2 *>(brow[r] + k0)));
                    b0 = bf.x * LOG2E; b1 = bf.y * LOG2E;
                } else if (BIAS_MODE == 2) {
                    const int2 kk = *reinterpret_cast<const int2 *>(kof + 8 * c + 2 * t);
                    b0 = k0 == 0 ? rp_k0[r] : sub[rp_base[r] - rp_mult[r] * kk.x];
                    b1 = sub[rp_base[r] - rp_mult[r] * kk.y];
                }
                float u0 = fmaf(sc[4 * c + 2 * r], p.scale_log2e, b0), u1 = fmaf(sc[4 * c + 2 * r + 1], p.scale_log2e, b1);
                u0 = k0 < p.N ? u0 : -INFINITY;
                u1 = k0 + 1 < p.N ? u1 : -INFINITY;
                sc[4 * c + 2 * r] = u0; sc[4 * c + 2 * r + 1] = u1;
                mx[r] = fmaxf(mx[r], fmaxf(u0, u1));
            }
        }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);      // every tile holds at least one valid key: finite
            alpha[r] = ex2_approx(m_run[r] - m_new);
            m_run[r] = m_new;
        }
        // ---- p = 2^(u - m) -> fp16 A fragments; the row sum adds the ROUNDED values, so the weights of a row sum to one -----
        uint32_t pa[AT_BKV / 16][4];
        float ls[2] = {0.f, 0.f};
#pragma unroll
        for (int c = 0; c < AT_BKV / 8; ++c) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float e0 = ex2_approx(sc[4 * c + 2 * r] - m_run[r]), e1 = ex2_approx(sc[4 * c + 2 * r + 1] - m_run[r]);
                const __half2 h2 = __floats2half2_rn(e0, e1);
                const float2 pr = __half22float2(h2);
                ls[r] += pr.x + pr.y;
                pa[c >> 1][(c & 1) * 2 + r] = *reinterpret_cast<const uint32_t *>(&h2);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = fmaf(l_run[r], alpha[r], ls[r]);
#pragma unroll
        for (int c = 0; c < AT_D / 8; ++c) { o[4 * c] *= alpha[0]; o[4 * c + 1] *= alpha[0]; o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1]; }
        // ---- O += P V_j ------------------------------------------------------------------------------------------------
        const uint32_t sv = smem_u32(sV + s * AT_KV_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_BKV / 16; ++k) wgmma_rs_n64_bt(o, pa[k], make_desc_mnmajor_sw128(sv + k * 16 * 128));
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&kv_empty[s]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (!q_ok[r]) continue;
        const float inv = 1.0f / l;
        __half *dst = p.out + (size_t)(row_base + qi[r]) * p.C + h * AT_D + 2 * t;
#pragma unroll
        for (int c = 0; c < AT_D / 8; ++c)
            *reinterpret_cast<__half2 *>(dst + 8 * c) = __floats2half2_rn(o[4 * c + 2 * r] * inv, o[4 * c + 2 * r + 1] * inv);
    }
}

template <int MODE>
static int launch_attn(const CUtensorMap &tm, const AttnParams &p, cudaStream_t stream) {
    const size_t tab = MODE == 2 ? (size_t)AT_STAGES * ((size_t)p.sub_stride * 4 + AT_BKV * 4) : 0;
    if (AT_TAB_OFF + tab > (size_t)AT_SMEM_MAX) { set_error("attention: relative-position window %d x %d too wide for the table sub-windows", p.gh, p.gw); return DM_E_UNSUPPORTED; }
    static PerDeviceFlag configured;
    if (!configured.test_and_set())
        DM_CUDA_CHECK(cudaFuncSetAttribute(attention_wgmma_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM_MAX));
    dim3 grid((p.N + AT_BQ - 1) / AT_BQ, p.H, p.B);
    attention_wgmma_kernel<MODE><<<grid, AT_THREADS, AT_TAB_OFF + tab, stream>>>(tm, p);
    DM_LAUNCH_CHECK("attention_wgmma_kernel");
    return DM_OK;
}

int attention_f16(const __half *qkv, AttnParams p, cudaStream_t stream, const float *rel_table = nullptr, int nrd = 0, int gh = 0, int gw = 0) {
    if (p.C != p.H * AT_D) { set_error("attention_f16: head_dim must be 64"); return DM_E_UNSUPPORTED; }
    CUtensorMap tm;
    int rc = make_tmap_2d(&tm, qkv, (uint64_t)p.B * p.N, (uint64_t)3 * p.C, (uint64_t)3 * p.C, AT_BQ, AT_D);
    if (rc) return rc;
    if (p.bias && (p.bias_ld % 8 != 0 || p.bias_ld < ((p.N + AT_BKV - 1) / AT_BKV) * AT_BKV)) {
        set_error("attention_f16: bias row pitch must be a multiple of 8 and cover whole 128-key tiles (got %d)", p.bias_ld);
        return DM_E_INVALID;
    }
    p.rel_table = rel_table; p.nrd = nrd; p.gh = gh; p.gw = gw; p.sub_stride = 0;
    if (rel_table) {
        if (gh < 1 || gw < 1 || (long long)gh * gw + 1 != p.N || (long long)nrd != (long long)(2 * gh - 1) * (2 * gw - 1) + 3) {
            set_error("attention_f16: relative-position mode needs N = gh*gw+1 and nrd = (2gh-1)(2gw-1)+3");
            return DM_E_INVALID;
        }
        p.sub_stride = relpos_sub_stride(gh, gw);
        return launch_attn<2>(tm, p, stream);
    }
    return p.bias ? launch_attn<1>(tm, p, stream) : launch_attn<0>(tm, p, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Split attention (the fp32-class path of no_half, bias mode 0): qkv is a split tensor [B*N, 9C], each row [hi | lo | hi] of the
// 3C-wide q, k, v; the output is split [B*N, 3C].  Same skeleton as above, with hi and lo tiles of Q, K and V in shared memory
// (160 KB).  Per KV tile:
//   S = Q_lo K_hi^T + Q_hi K_lo^T + Q_hi K_hi^T   twelve m64n128k16: the small cross terms go first, so the accumulator's
//                                                 alignment truncation only acts at the magnitude of S for the last four
//   fp32 online softmax; p = 2^(u - m) * 2^12 split into p_hi + p_lo (the 2^12 keeps p_lo out of the fp16 subnormals for
//   p > 2^-15; it cancels against the row sum, which adds the same unsplit fp32 values)
//   PV = P_lo V_hi + P_hi V_lo + P_hi V_hi     twenty-four m64n64k16 into a FRESH accumulator, then O = O * alpha + PV by FFMA,
//                                              so the running O never sits in a truncating accumulator across KV tiles
// ---------------------------------------------------------------------------------------------------------------------
constexpr int AS_K_OFF = 2 * AT_Q_BYTES;                          // Q hi | Q lo, then per stage K hi | K lo, then V hi | V lo
constexpr int AS_V_OFF = AS_K_OFF + AT_STAGES * 2 * AT_KV_BYTES;
constexpr int AS_BAR_OFF = AS_V_OFF + AT_STAGES * 2 * AT_KV_BYTES;
constexpr int AS_SMEM = AS_BAR_OFF + 64;

__global__ void __launch_bounds__(AT_THREADS, 1) attention_split_kernel(const __grid_constant__ CUtensorMap tmQKV, AttnParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *sQ = smem_raw, *sK = smem_raw + AS_K_OFF, *sV = smem_raw + AS_V_OFF;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + AS_BAR_OFF);
    uint64_t *q_full = bars, *kv_full = bars + 1, *kv_empty = bars + 1 + AT_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ, h = blockIdx.y, b = blockIdx.z;
    const int num_kv = (p.N + AT_BKV - 1) / AT_BKV;
    const int row_base = b * p.N;
    const int lo = 3 * p.C;                   // column offset of the lo halves in a qkv row

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmQKV);
        mbar_init(q_full, 1);
        for (int s = 0; s < AT_STAGES; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(q_full, 2 * AT_Q_BYTES);
            tma_load_2d(sQ, &tmQKV, q_full, h * AT_D, row_base + q0);
            tma_load_2d(sQ + AT_Q_BYTES, &tmQKV, q_full, lo + h * AT_D, row_base + q0);
            for (int j = 0; j < num_kv; ++j) {
                const int s = j % AT_STAGES, r = row_base + j * AT_BKV;
                uint8_t *k = sK + s * 2 * AT_KV_BYTES, *v = sV + s * 2 * AT_KV_BYTES;
                mbar_wait(&kv_empty[s], ((j / AT_STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(&kv_full[s], 4 * AT_KV_BYTES);
                tma_load_2d(k, &tmQKV, &kv_full[s], p.C + h * AT_D, r);
                tma_load_2d(k + AT_KV_BYTES, &tmQKV, &kv_full[s], lo + p.C + h * AT_D, r);
                tma_load_2d(v, &tmQKV, &kv_full[s], 2 * p.C + h * AT_D, r);
                tma_load_2d(v + AT_KV_BYTES, &tmQKV, &kv_full[s], lo + 2 * p.C + h * AT_D, r);
            }
        }
        return;
    }

    const int wg = (warp >> 2) - 1, t = lane & 3;
    int qi[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) qi[r] = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint64_t qh_desc = make_desc_kmajor_sw128(smem_u32(sQ) + wg * (64 * 128));
    const uint64_t ql_desc = make_desc_kmajor_sw128(smem_u32(sQ + AT_Q_BYTES) + wg * (64 * 128));

    mbar_wait(q_full, 0);
    for (int j = 0; j < num_kv; ++j) {
        const int s = j % AT_STAGES;
        const int kbase = j * AT_BKV;
        mbar_wait(&kv_full[s], (j / AT_STAGES) & 1);
        float sc[64];
        const uint32_t sk = smem_u32(sK + s * 2 * AT_KV_BYTES);
        const uint64_t kh_desc = make_desc_kmajor_sw128(sk), kl_desc = make_desc_kmajor_sw128(sk + AT_KV_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_ss<AT_BKV>(sc, ql_desc + (uint64_t)(2 * k), kh_desc + (uint64_t)(2 * k), k != 0);
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_ss<AT_BKV>(sc, qh_desc + (uint64_t)(2 * k), kl_desc + (uint64_t)(2 * k), 1);
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_ss<AT_BKV>(sc, qh_desc + (uint64_t)(2 * k), kh_desc + (uint64_t)(2 * k), 1);
        wgmma_commit();
        wgmma_wait<0>();
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int c = 0; c < AT_BKV / 8; ++c) {
            const int k0 = kbase + 8 * c + 2 * t;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float u0 = sc[4 * c + 2 * r] * p.scale_log2e, u1 = sc[4 * c + 2 * r + 1] * p.scale_log2e;
                u0 = k0 < p.N ? u0 : -INFINITY;
                u1 = k0 + 1 < p.N ? u1 : -INFINITY;
                sc[4 * c + 2 * r] = u0; sc[4 * c + 2 * r + 1] = u1;
                mx[r] = fmaxf(mx[r], fmaxf(u0, u1));
            }
        }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            alpha[r] = ex2_approx(m_run[r] - m_new);
            m_run[r] = m_new;
        }
        uint32_t ph[AT_BKV / 16][4], pl[AT_BKV / 16][4];
        float ls[2] = {0.f, 0.f};
#pragma unroll
        for (int c = 0; c < AT_BKV / 8; ++c) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float e0 = ex2_approx(sc[4 * c + 2 * r] - m_run[r]) * 4096.f, e1 = ex2_approx(sc[4 * c + 2 * r + 1] - m_run[r]) * 4096.f;
                ls[r] += e0 + e1;
                const __half2 hi = __floats2half2_rn(e0, e1);
                const float2 hf = __half22float2(hi);
                const __half2 lo2 = __floats2half2_rn(e0 - hf.x, e1 - hf.y);
                ph[c >> 1][(c & 1) * 2 + r] = *reinterpret_cast<const uint32_t *>(&hi);
                pl[c >> 1][(c & 1) * 2 + r] = *reinterpret_cast<const uint32_t *>(&lo2);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = fmaf(l_run[r], alpha[r], ls[r]);
        float pv[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) pv[i] = 0.f;
        const uint32_t sv = smem_u32(sV + s * 2 * AT_KV_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_BKV / 16; ++k) wgmma_rs_n64_bt(pv, pl[k], make_desc_mnmajor_sw128(sv + k * 16 * 128));
#pragma unroll
        for (int k = 0; k < AT_BKV / 16; ++k) wgmma_rs_n64_bt(pv, ph[k], make_desc_mnmajor_sw128(sv + AT_KV_BYTES + k * 16 * 128));
#pragma unroll
        for (int k = 0; k < AT_BKV / 16; ++k) wgmma_rs_n64_bt(pv, ph[k], make_desc_mnmajor_sw128(sv + k * 16 * 128));
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&kv_empty[s]);
#pragma unroll
        for (int c = 0; c < AT_D / 8; ++c) {
            o[4 * c] = fmaf(o[4 * c], alpha[0], pv[4 * c]); o[4 * c + 1] = fmaf(o[4 * c + 1], alpha[0], pv[4 * c + 1]);
            o[4 * c + 2] = fmaf(o[4 * c + 2], alpha[1], pv[4 * c + 2]); o[4 * c + 3] = fmaf(o[4 * c + 3], alpha[1], pv[4 * c + 3]);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (qi[r] >= p.N) continue;
        __half *dst = p.out + (size_t)(row_base + qi[r]) * (3 * p.C) + h * AT_D + 2 * t;
#pragma unroll
        for (int c = 0; c < AT_D / 8; ++c) {
            const float v0 = o[4 * c + 2 * r] / l, v1 = o[4 * c + 2 * r + 1] / l;
            const __half2 hi = __floats2half2_rn(v0, v1);
            const float2 hf = __half22float2(hi);
            *reinterpret_cast<__half2 *>(dst + 8 * c) = hi;
            *reinterpret_cast<__half2 *>(dst + p.C + 8 * c) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
            *reinterpret_cast<__half2 *>(dst + 2 * p.C + 8 * c) = hi;
        }
    }
}

int attention_split(const __half *qkv, AttnParams p, cudaStream_t stream) {
    if (p.C != p.H * AT_D || p.H < 1) { set_error("dm_attention_split: head_dim must be 64"); return DM_E_UNSUPPORTED; }
    if (p.N < 2 || p.B < 1 || !qkv || !p.out) { set_error("dm_attention_split: bad arguments (N >= 2 tokens, B >= 1)"); return DM_E_INVALID; }
    CUtensorMap tm;
    int rc = make_tmap_2d(&tm, qkv, (uint64_t)p.B * p.N, (uint64_t)9 * p.C, (uint64_t)9 * p.C, AT_BQ, AT_D);
    if (rc) return rc;
    static PerDeviceFlag configured;
    if (!configured.test_and_set())
        DM_CUDA_CHECK(cudaFuncSetAttribute(attention_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM));
    dim3 grid((p.N + AT_BQ - 1) / AT_BQ, p.H, p.B);
    attention_split_kernel<<<grid, AT_THREADS, AS_SMEM, stream>>>(tm, p);
    DM_LAUNCH_CHECK("attention_split_kernel");
    return DM_OK;
}

}  // namespace dm

extern "C" __attribute__((visibility("default"))) int dm_attention_split(const void *qkv, int B, int N, int H, float scale, void *out, void *stream) {
    dm::AttnParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.N = N; p.H = H; p.C = H * 64;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.out = (__half *)out;
    return dm::attention_split((const __half *)qkv, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_attention_f16(const void *qkv, int B, int N, int H, float scale, const void *bias, int bias_ld,
                                                                    void *out, void *stream) {
    dm::AttnParams p;
    p.B = B; p.N = N; p.H = H; p.C = H * 64;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.bias = (const __half *)bias; p.bias_ld = bias_ld;
    p.out = (__half *)out;
    return dm::attention_f16((const __half *)qkv, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_attention_relpos_f16(const void *qkv, int B, int gh, int gw, int H, float scale,
                                                                           const float *rel_table_log2e, int nrd,
                                                                           void *out, void *stream) {
    dm::AttnParams p;
    p.B = B; p.N = gh * gw + 1; p.H = H; p.C = H * 64;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.bias = nullptr; p.bias_ld = 0;
    p.out = (__half *)out;
    if (!rel_table_log2e) { dm::set_error("dm_attention_relpos_f16: table is NULL"); return DM_E_INVALID; }
    return dm::attention_f16((const __half *)qkv, p, (cudaStream_t)stream, rel_table_log2e, nrd, gh, gw);
}
