// Tensor-core GEMM / implicit-GEMM convolution for sm_90a: C[M,N] = A[M,K] * W[N,K]^T with fused epilogues.
//
// Used for every Linear layer of the ViT (QKV, proj, fc1, fc2 — reference: timm Block / dinov2_layers/{attention,mlp}.py),
// the patch embedding, the DPT 1x1 convs, ConvTranspose k=s layers (GEMM + pixel-shuffle store) and, with CONV=true,
// the 3x3 stride-1 pad-1 convolutions of the DPT decoder (reference: dmidas/blocks.py, depth_anything_v2/util/blocks.py)
// as implicit GEMM over NHWC activations: the 9 taps are 9 shifted TMA boxes, zero padding = TMA out-of-bounds fill.
// Circular padding (tiling mode) reads a copy of the activations with a one-pixel wrapped border instead (conv_halo_circular).
//
// Structure (persistent, warp-specialised, ping-pong; one CTA of three warpgroups per SM):
//   the grid is min(tiles, SMs); CTA b walks tiles b, b + grid, ... of one static order (launch_gemm: groups of m-tiles,
//   n fastest inside a group, so the weight panels stay in L2 and each activation panel is read from HBM once)
//   warpgroup 0   : TMA producer — drops to 40 registers (setmaxnreg); one thread issues cp.async.bulk.tensor for every
//                   k-block of every tile of the CTA, in order, into one STAGES-deep ring of 128B-swizzled smem tiles
//                   (mbarrier tx), running ahead across tile boundaries
//   warpgroups 1-2: consumers — limit raised to 232 registers (the kernel builds in 168); each owns a whole BM x BN output tile and the two take alternate
//                   tiles of the CTA's sequence (so alternate runs of the ring).  wgmma.mma_async m64nBNk16, BM / 64 per
//                   16-wide k-slice (fp16 operands from shared memory, fp32 accumulators in registers), one commit group per
//                   k-block, the previous k-block's ring slot released once its group has retired.  A pair of named
//                   barriers makes the two main loops alternate: a warpgroup hands the tensor cores over as soon as its
//                   last MMA is issued and runs its epilogue under the other's main loop.  The epilogue works on the
//                   accumulator fragment: bias / GELU / ReLU / LayerScale+residual / pixel-shuffle / fused 1x1 head,
//                   8-byte (fp32) or 4-byte (fp16) accesses in which the four lanes of a quad cover one 32- or 16-byte run
//                   of a row
// Every output element sums the same k-blocks and 16-wide k-slices in the same order whatever the tile shape or schedule,
// so the results do not depend on either.
//
// Split mode (gemm_split / conv3x3_split, the fp32-class path of no_half): an fp32 activation a is stored as fp16 a_hi =
// rn(a), a_lo = rn(a - a_hi) in one tensor of 3x the width, each row [a_hi | a_lo | a_hi]; the weights are packed
// [w_hi | w_hi | w_lo] after a per-output-channel power-of-two pre-scale (so the low halves stay normal), and the MMA over the
// tripled depth forms a_hi w_hi + a_lo w_hi + a_hi w_lo.  The tensor core's fp32 accumulator aligns and truncates its partial
// sums (tools/probe_tensor_core.py), a bias that grows with the number of k-steps accumulated in it, so the split mainloop
// PROMOTES: every SPLIT_PROMOTE k-blocks it waits for its MMAs, adds the wgmma accumulator into a register-resident fp32 sum with
// rounding FADDs and restarts the accumulator.  SPLIT_PROMOTE = 1 (64 of the tripled depth, four k-steps), chosen by measurement
// (tools/probe_tensor_core.py's method, H100 SXM 80 GB at 700 W): with all-positive products the relative bias of the split GEMM
// is -1.4e-7 at P = 1, -3.8e-7 at 2, -1.0e-6 at 4 and -5.3e-6 at 16 k-blocks, independent of K (fp32 torch.matmul: 1e-9); its
// largest error on random-sign data is 2.6-4.6x fp32's at P = 1, 2.2-2.9x at P = 4 and up to 8.2x at P = 16 (K = 1024 to
// 49152); and P = 1 was also the fastest in that one run (ViT-L batch-32 fc2 / fc1 / qkv: 423 / 299 / 322 TFLOP/s of MMA work,
// against 369 / 293 / 306 at P = 4).  The extra fp32 sum doubles the accumulator registers, so split tiles are 128 x 64 (or
// 128 x 32): 168 registers, no spills.
// Split epilogues undo the pre-scale, apply bias / activation / residual in fp32 and store split outputs (or fp32 ones).
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dm {
using namespace tc;

enum GemmEpi : int {
    EPI_STORE_F16 = 0,   // C = act(acc + bias) [+ R]           -> fp16 [M, ldc]   (+ optional relu copy C2)
    EPI_RESID_F32 = 1,   // X += gamma[n] * (acc + bias[n])     -> fp32 in place (LayerScale + residual)
    EPI_PIXSHUF = 2,     // ConvTranspose k=s: n = (i, j, co) scattered to out[b, s*y+i, s*x+j, co]
    EPI_HEAD = 3,        // relu(acc + bias) . w2 + b2 -> relu -> fp32 [M]   (conv3x3 -> ReLU -> conv1x1 -> ReLU fused; BN = N)
    EPI_STORE_F32 = 4,   // C = acc + bias -> fp32 [M, ldc]
};
enum GemmAct : int { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };

struct GemmParams {
    int M, N, K;
    int epi, act;
    const float *bias;      // [N] or null
    __half *C; int ldc;     // fp16 output
    __half *C2;             // optional relu(C) copy (same layout) or null
    const __half *R; int ldr;  // optional fp16 residual added before the store (EPI_STORE_F16)
    const __half *R2; int ldr2;  // optional second fp16 residual
    float *X; int ldx;      // fp32 residual stream (EPI_RESID_F32) / fp32 output (EPI_STORE_F32, EPI_HEAD)
    const float *gamma;     // [N] LayerScale (EPI_RESID_F32) / w2 (EPI_HEAD)
    float head_b2;
    // pixel shuffle
    int ps_s, ps_cout, ps_h, ps_w;
    // implicit conv geometry (CONV): activations [B, H, W, Cin]; tile = hbox x wbox pixels
    int cB, cH, cW, cCin, hbox, wbox, tiles_x, tiles_y;
    // static tile schedule (launch_gemm)
    int m_tiles, n_tiles, group_m;
    // implicit conv: tap offset into the tensor map, 0 = the activations themselves, 1 = their [B, H+2, W+2, Cin] halo copy (circular
    // padding).  Last, so that the other fields keep their offsets and the plain GEMM kernels their code
    int corg;
    // split mode: [N] fp32 factor undoing the weights' power-of-two pre-scale
    const float *wscale;
};

// BM x BN = the output tile of ONE consumer warpgroup.  The ring takes what the 227 KB of shared memory allows, up to 8
// stages: 6 x 32 KB for 128 x 128, 5 x 40 KB for 64 x 256.
template <int BM, int BN>
struct GemmCfg {
    static constexpr int BK = 64;
    static constexpr int WM = BM / 64;                  // m64nBNk16 per k-slice
    static constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (220 * 1024) / STAGE_BYTES < 8 ? (220 * 1024) / STAGE_BYTES : 8;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 /*barriers*/;   // base is __align__(1024)
};
constexpr int GEMM_THREADS = 384;
constexpr int SPLIT_PROMOTE = 1;    // split mode: k-blocks per wgmma accumulator before it is added into the fp32 sum (header)

// exact-erf GELU, one MUFU.  With u = min(|x|, 5.75):
//     gelu(x) = max(x, 0) - u * 2^(-u Q(u) - 1),      Q(u) = -log2(erfc(u / sqrt 2)) / u
// Q is smooth and nearly linear on [0, 5.75]; the degree-5 fit below (Lawson-weighted on the GELU error) keeps
// |gelu - x Phi(x)| < 3.2e-7 in fp32 over all x (tests/test_gelu_formula.py checks the same numbers on
// the host), i.e. three orders below the fp16 rounding of the stored activation.  Past the clamp u*2^(..) < 3e-8.
__device__ __forceinline__ float gelu_erf(float x) {
    const float u = fminf(fabsf(x), 5.75f);
    float q = -2.992472582263872e-05f;
    q = fmaf(q, u, 0.0007398786256089807f);
    q = fmaf(q, u, -0.007977476343512535f);
    q = fmaf(q, u, 0.05323820561170578f);
    q = fmaf(q, u, 0.45891568064689636f);
    q = fmaf(q, u, 1.1511471271514893f);
    float e;
    const float t = fmaf(-u, q, -1.f);
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
    return fmaf(-u, e, fmaxf(x, 0.f));
}

// (v0, v1) as split fp16 pairs: hi at dst, lo at dst + lo_off, hi again at dst + 2 lo_off
__device__ __forceinline__ void split_store2(__half *dst, int lo_off, float v0, float v1) {
    const __half2 hi = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    *reinterpret_cast<__half2 *>(dst) = hi;
    *reinterpret_cast<__half2 *>(dst + lo_off) = lo;
    *reinterpret_cast<__half2 *>(dst + 2 * lo_off) = hi;
}

// Epilogue of one consumer thread: its accumulator fragment holds rows r0 = 16 * warp + lane / 4 and r0 + 8 of the
// warpgroup's 64, and for every 8-column group j the columns 8j + 2 (lane % 4), +1 (tc_common.cuh).  EPI = p.epi, fixed at
// compile time so that a tile's epilogue is only the code of its own mode: the fully unrolled epilogue of all modes is
// larger than the instruction cache and would otherwise be streamed through it under the other warpgroup's main loop.
// SPLIT: the operands R / R2 are split tensors (lo halves p.N columns after the hi ones), the output is stored split (C,
// C2: [hi | lo | hi] at column offsets 0, N, 2N; pixel shuffle: per output pixel, offsets 0, cout, 2 cout) and the
// accumulator is multiplied by wscale[n] first.
template <int BN, int EPI, bool SPLIT = false>
__device__ __forceinline__ void epilogue_fragment(const GemmParams &p, const float (&acc)[BN / 2], const long long (&m)[2], const bool (&row_ok)[2],
                                                  int n_base, int lane) {
    // Column groups are taken JC at a time: every operand load of a chunk is issued before its first store, so the loads
    // of a chunk are in flight together instead of each waiting behind the previous group's store (X is read and written).
    constexpr int JC = 2;
    const int t = lane & 3;
    float head_acc[2] = {0.f, 0.f};
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += JC) {
        float2 b2[JC], g2[JC], x[JC][2], ws[JC];
        __half2 rv[JC][2], rv2[JC][2], rl[JC][2], rl2[JC][2];
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
            const int n = n_base + 8 * (j0 + jj) + 2 * t;
            b2[jj] = make_float2(0.f, 0.f);
            g2[jj] = make_float2(0.f, 0.f);
            if (n >= p.N) continue;
            if (p.bias) b2[jj] = __ldg(reinterpret_cast<const float2 *>(p.bias + n));
            if (SPLIT) ws[jj] = __ldg(reinterpret_cast<const float2 *>(p.wscale + n));
            if (EPI == EPI_RESID_F32 || EPI == EPI_HEAD) g2[jj] = __ldg(reinterpret_cast<const float2 *>(p.gamma + n));
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!row_ok[r]) continue;
                if (EPI == EPI_RESID_F32) x[jj][r] = *reinterpret_cast<const float2 *>(p.X + m[r] * p.ldx + n);
                if (EPI == EPI_STORE_F16 || EPI == EPI_PIXSHUF) {
                    if (p.R) rv[jj][r] = __ldg(reinterpret_cast<const __half2 *>(p.R + m[r] * p.ldr + n));
                    if (p.R2) rv2[jj][r] = __ldg(reinterpret_cast<const __half2 *>(p.R2 + m[r] * p.ldr2 + n));
                    if (SPLIT && p.R) rl[jj][r] = __ldg(reinterpret_cast<const __half2 *>(p.R + m[r] * p.ldr + p.N + n));
                    if (SPLIT && p.R2) rl2[jj][r] = __ldg(reinterpret_cast<const __half2 *>(p.R2 + m[r] * p.ldr2 + p.N + n));
                }
            }
        }
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
            const int j = j0 + jj;
            const int n = n_base + 8 * j + 2 * t;
            if (n >= p.N) continue;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!row_ok[r]) continue;
                float v0, v1;
                if (SPLIT) { v0 = fmaf(acc[4 * j + 2 * r], ws[jj].x, b2[jj].x); v1 = fmaf(acc[4 * j + 2 * r + 1], ws[jj].y, b2[jj].y); }
                else { v0 = acc[4 * j + 2 * r] + b2[jj].x; v1 = acc[4 * j + 2 * r + 1] + b2[jj].y; }
                if (EPI == EPI_RESID_F32) {
                    float2 xv = x[jj][r];
                    xv.x = fmaf(g2[jj].x, v0, xv.x); xv.y = fmaf(g2[jj].y, v1, xv.y);
                    *reinterpret_cast<float2 *>(p.X + m[r] * p.ldx + n) = xv;
                    continue;
                }
                if (EPI == EPI_STORE_F32) {
                    *reinterpret_cast<float2 *>(p.X + m[r] * p.ldx + n) = make_float2(v0, v1);
                    continue;
                }
                if (p.act == ACT_GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
                else if (p.act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (EPI == EPI_HEAD) {
                    head_acc[r] = fmaf(v1, g2[jj].y, fmaf(v0, g2[jj].x, head_acc[r]));
                    continue;
                }
                if (SPLIT) {
                    if (p.R) { const float2 f = __half22float2(rv[jj][r]), l = __half22float2(rl[jj][r]); v0 += f.x + l.x; v1 += f.y + l.y; }
                    if (p.R2) { const float2 f = __half22float2(rv2[jj][r]), l = __half22float2(rl2[jj][r]); v0 += f.x + l.x; v1 += f.y + l.y; }
                    __half *dst;
                    int lo_off;
                    if (EPI == EPI_PIXSHUF) {
                        const int s = p.ps_s, ij = n / p.ps_cout, co = n % p.ps_cout;
                        const int i = ij / s, jx = ij % s;
                        const long long bb = m[r] / ((long long)p.ps_h * p.ps_w);
                        const int rem = (int)(m[r] % ((long long)p.ps_h * p.ps_w));
                        const int y = rem / p.ps_w, xx = rem % p.ps_w;
                        dst = p.C + (((bb * (p.ps_h * s) + (y * s + i)) * (long long)(p.ps_w * s)) + (xx * s + jx)) * (3 * p.ps_cout) + co;
                        lo_off = p.ps_cout;
                    } else {
                        dst = p.C + m[r] * p.ldc + n;
                        lo_off = p.N;
                    }
                    split_store2(dst, lo_off, v0, v1);
                    if (EPI != EPI_PIXSHUF && p.C2) split_store2(p.C2 + m[r] * p.ldc + n, lo_off, fmaxf(v0, 0.f), fmaxf(v1, 0.f));
                    continue;
                }
                if (p.R) { const float2 f = __half22float2(rv[jj][r]); v0 += f.x; v1 += f.y; }
                if (p.R2) { const float2 f = __half22float2(rv2[jj][r]); v0 += f.x; v1 += f.y; }
                const __half2 h2 = __floats2half2_rn(v0, v1);
                if (EPI == EPI_PIXSHUF) {
                    const int s = p.ps_s, ij = n / p.ps_cout, co = n % p.ps_cout;
                    const int i = ij / s, jx = ij % s;
                    const long long bb = m[r] / ((long long)p.ps_h * p.ps_w);
                    const int rem = (int)(m[r] % ((long long)p.ps_h * p.ps_w));
                    const int y = rem / p.ps_w, xx = rem % p.ps_w;
                    *reinterpret_cast<__half2 *>(p.C + (((bb * (p.ps_h * s) + (y * s + i)) * (long long)(p.ps_w * s)) + (xx * s + jx)) * p.ps_cout + co) = h2;
                } else {
                    *reinterpret_cast<__half2 *>(p.C + m[r] * p.ldc + n) = h2;
                    if (p.C2) *reinterpret_cast<__half2 *>(p.C2 + m[r] * p.ldc + n) = __hmax2(h2, __float2half2_rn(0.f));
                }
            }
        }
    }
    if (EPI == EPI_HEAD) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float s = head_acc[r];
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            if (t == 0 && row_ok[r]) p.X[m[r]] = fmaxf(s + p.head_b2, 0.f);
        }
    }
}

// tile t of the static schedule -> (m tile, n tile): groups of group_m m-tiles, n fastest inside a group (see launch_gemm)
__device__ __forceinline__ void tile_coords(const GemmParams &p, int t, int &m_blk, int &n_blk) {
    const int per_group = p.group_m * p.n_tiles;
    const int g = t / per_group, r = t - g * per_group;
    m_blk = g * p.group_m + r / p.n_tiles;
    n_blk = r % p.n_tiles;
}

// implicit conv: m tile -> (image, top row, left column) of its hbox x wbox pixel box
__device__ __forceinline__ void conv_origin(const GemmParams &p, int m_blk, int &cb, int &cy0, int &cx0) {
    const int tiles_per_img = p.tiles_x * p.tiles_y;
    cb = m_blk / tiles_per_img;
    const int t = m_blk % tiles_per_img;
    cy0 = (t / p.tiles_x) * p.hbox;
    cx0 = (t % p.tiles_x) * p.wbox;
}

template <int BM, int BN, bool CONV, bool SPLIT>
__device__ __forceinline__ void gemm_body(const CUtensorMap &tmA, const CUtensorMap &tmB, const GemmParams &p) {
    using Cfg = GemmCfg<BM, BN>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = smem_raw;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
    uint64_t *empty = full + Cfg::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = CONV ? 9 * (p.cCin / Cfg::BK) : p.K / Cfg::BK;
    const int my_tiles = (p.m_tiles * p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // grid <= tiles: >= 1

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }   // the 4 warps of one consumer
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            // one ring across the CTA's whole tile sequence: tile i's k-blocks follow tile i-1's
            int stage = 0, phase = 0;
            for (int i = 0; i < my_tiles; ++i) {
                int m_blk, n_blk, cb = 0, cy0 = 0, cx0 = 0;
                tile_coords(p, blockIdx.x + i * gridDim.x, m_blk, n_blk);
                if (CONV) conv_origin(p, m_blk, cb, cy0, cx0);
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t *sa = smem + stage * Cfg::STAGE_BYTES, *sb = sa + Cfg::A_BYTES;
                    mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
                    if (CONV) {
                        const int cblks = p.cCin / Cfg::BK;
                        const int tap = kb / cblks, cblk = kb % cblks;
                        const int dy = tap / 3 - 1, dx = tap % 3 - 1;
                        tma_load_4d(sa, &tmA, &full[stage], cblk * Cfg::BK, cx0 + dx + p.corg, cy0 + dy + p.corg, cb);
                    } else {
                        tma_load_2d(sa, &tmA, &full[stage], kb * Cfg::BK, m_blk * BM);
                    }
                    tma_load_2d(sb, &tmB, &full[stage], kb * Cfg::BK, n_blk * BN);
                    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg takes tiles wg, wg + 2, ... of the CTA's sequence, each a whole BM x BN tile =====
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    float acc[Cfg::WM][BN / 2];
    float sum[Cfg::WM][BN / 2];      // split mode: the promoted fp32 sum (unused otherwise)
    for (int i = wg; i < my_tiles; i += 2) {
        int m_blk, n_blk, cb = 0, cy0 = 0, cx0 = 0;
        tile_coords(p, blockIdx.x + i * gridDim.x, m_blk, n_blk);
        if (CONV) conv_origin(p, m_blk, cb, cy0, cx0);
        const long long q0 = (long long)i * num_kb;              // ring position of the tile's first k-block
        int stage = (int)(q0 % Cfg::STAGES), phase = (int)((q0 / Cfg::STAGES) & 1), prev = 0;
        // ping-pong: the main loops of the two warpgroups alternate, so one's epilogue runs under the other's MMAs.  The
        // alternation is also what makes the parity waits below sound: every ring position before q0 has already been
        // waited for, so no full barrier is more than one phase behind this warpgroup's wait.
        if (i > 0) named_bar_sync(1 + wg, 256);
        if (SPLIT) {
#pragma unroll
            for (int h = 0; h < Cfg::WM; ++h)
#pragma unroll
                for (int e = 0; e < BN / 2; ++e) sum[h][e] = 0.f;
        }
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES), sb = sa + Cfg::A_BYTES;
            const uint64_t bdesc = make_desc_kmajor_sw128(sb);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < Cfg::BK / 16; ++k) {
#pragma unroll
                for (int h = 0; h < Cfg::WM; ++h)
                    wgmma_ss<BN>(acc[h], make_desc_kmajor_sw128(sa + h * (64 * 128)) + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k),
                                 SPLIT ? ((kb % SPLIT_PROMOTE) | k) != 0 : (kb | k) != 0);
            }
            wgmma_commit();
            if (kb > 0) {                       // the previous k-block's MMAs have retired: hand its slot back to the producer
                wgmma_wait<1>();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            if (SPLIT && ((kb + 1) % SPLIT_PROMOTE == 0 || kb + 1 == num_kb)) {   // promotion: fp32 sum += accumulator
                wgmma_wait<0>();
#pragma unroll
                for (int h = 0; h < Cfg::WM; ++h)
#pragma unroll
                    for (int e = 0; e < BN / 2; ++e) sum[h][e] = __fadd_rn(sum[h][e], acc[h][e]);
            }
            prev = stage;
            if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        if (i + 1 < my_tiles) named_bar_arrive(2 - wg, 256);   // all MMAs issued: the other warpgroup's main loop may start
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&empty[prev]);

#pragma unroll
        for (int h = 0; h < Cfg::WM; ++h) {
            long long m[2];
            bool row_ok[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = h * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
                if (CONV) {
                    const int y = cy0 + row / p.wbox, x = cx0 + row % p.wbox;
                    row_ok[r] = (y < p.cH) && (x < p.cW);
                    m[r] = ((long long)cb * p.cH + y) * p.cW + x;
                } else {
                    m[r] = (long long)m_blk * BM + row;
                    row_ok[r] = m[r] < p.M;
                }
            }
            const float (&res)[BN / 2] = SPLIT ? sum[h] : acc[h];
            switch (p.epi) {
                case EPI_STORE_F16: epilogue_fragment<BN, EPI_STORE_F16, SPLIT>(p, res, m, row_ok, n_blk * BN, lane); break;
                case EPI_RESID_F32: epilogue_fragment<BN, EPI_RESID_F32, SPLIT>(p, res, m, row_ok, n_blk * BN, lane); break;
                case EPI_PIXSHUF: epilogue_fragment<BN, EPI_PIXSHUF, SPLIT>(p, res, m, row_ok, n_blk * BN, lane); break;
                case EPI_HEAD: epilogue_fragment<BN, EPI_HEAD, SPLIT>(p, res, m, row_ok, n_blk * BN, lane); break;
                case EPI_STORE_F32: epilogue_fragment<BN, EPI_STORE_F32, SPLIT>(p, res, m, row_ok, n_blk * BN, lane); break;
            }
        }
    }
}

template <int BM, int BN, bool CONV>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmB, GemmParams p) {
    gemm_body<BM, BN, CONV, false>(tmA, tmB, p);
}

// split mode (header): promoted mainloop, split epilogues
template <int BM, int BN, bool CONV>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_split_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmB, GemmParams p) {
    gemm_body<BM, BN, CONV, true>(tmA, tmB, p);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
        fn = (PFN_encodeTiled)p;
    }
    return fn;
}

// 2-D fp16 row-major [rows, cols] with row pitch ld (elements); box = box_rows x 64 cols, 128B swizzle
int make_tmap_2d(CUtensorMap *tm, const void *ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return DM_E_CUDA; }
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(2d) failed: %d (rows=%llu cols=%llu ld=%llu)", (int)r, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld); return DM_E_CUDA; }
    return DM_OK;
}

// 4-D fp16 NHWC [B, H, W, C]; box = [1, hbox, wbox, 64]
int make_tmap_nhwc(CUtensorMap *tm, const void *ptr, uint64_t B, uint64_t H, uint64_t W, uint64_t C, uint32_t hbox, uint32_t wbox) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return DM_E_CUDA; }
    cuuint64_t dims[4] = {C, W, H, B};
    cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
    cuuint32_t box[4] = {64, wbox, hbox, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(4d) failed: %d", (int)r); return DM_E_CUDA; }
    return DM_OK;
}

// Tile order.  The CTAs running together cover about SMs consecutive tiles of the order.  With n fastest inside a group of
// group_m m-tiles, those tiles share a few activation panels (A, 32-268 MB at the trunk's shapes) and sweep the weight matrix
// (2-8 MB) across n; an activation panel is therefore read from HBM once and used for every n-tile while it is still in the
// 50 MB L2, and the weights stay L2-resident for the whole call.  group_m bounds the activation panels of a group plus the
// whole weight matrix by about half the L2 (the m fastest order re-read all of A once per weight panel).
template <int BM, int BN, bool CONV, bool SPLIT = false>
static int launch_gemm(const CUtensorMap &tmA, const CUtensorMap &tmB, GemmParams p, int m_tiles, cudaStream_t stream) {
    using Cfg = GemmCfg<BM, BN>;
    static PerDeviceFlag configured;
    static PerDeviceAttr sms(cudaDevAttrMultiProcessorCount);
    void (*kernel)(const CUtensorMap, const CUtensorMap, GemmParams);
    if constexpr (SPLIT) kernel = gemm_split_kernel<BM, BN, CONV>;
    else kernel = gemm_wgmma_kernel<BM, BN, CONV>;
    if (!configured.test_and_set())
        DM_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    const long long l2_budget = 24ll << 20, w_bytes = 2ll * p.N * p.K, a_panel = 2ll * BM * p.K;   // conv: K = 9 Cin over-counts
    const long long g = (l2_budget - w_bytes) / a_panel;
    p.m_tiles = m_tiles;
    p.n_tiles = (p.N + BN - 1) / BN;
    p.group_m = (int)(g < 1 ? 1 : (g > m_tiles ? m_tiles : g));
    const int tiles = m_tiles * p.n_tiles;
    const int grid = tiles < sms.get() ? tiles : sms.get();   // persistent: one CTA per SM, never more CTAs than tiles
    kernel<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, p);
    DM_LAUNCH_CHECK(SPLIT ? "gemm_split_kernel" : "gemm_wgmma_kernel");
    return DM_OK;
}

// The epilogue reads and writes column PAIRS: 8-byte accesses to the fp32 operands (bias, gamma, X), 4-byte ones to the fp16
// operands (C, C2, R, R2).  Their pitches must therefore be even and their base addresses aligned accordingly.
static int check_epilogue_operands(const GemmParams &p, const char *who) {
    auto misaligned = [](const void *q, size_t a) { return q && (reinterpret_cast<uintptr_t>(q) % a) != 0; };
    const bool f32_rows = p.epi == EPI_RESID_F32 || p.epi == EPI_STORE_F32;
    const bool f16_rows = p.epi == EPI_STORE_F16 || p.epi == EPI_PIXSHUF;
    if ((f32_rows && (!p.X || p.ldx % 2)) || (p.epi == EPI_HEAD && !p.X)) { set_error("%s: fp32 output missing or its pitch is odd (ldx=%d)", who, p.ldx); return DM_E_INVALID; }
    if (f16_rows && (!p.C || (p.epi == EPI_STORE_F16 && p.ldc % 2))) { set_error("%s: fp16 output missing or its pitch is odd (ldc=%d)", who, p.ldc); return DM_E_INVALID; }
    if (f16_rows && ((p.R && p.ldr % 2) || (p.R2 && p.ldr2 % 2))) { set_error("%s: residual pitches must be even (ldr=%d ldr2=%d)", who, p.ldr, p.ldr2); return DM_E_INVALID; }
    if (p.epi == EPI_PIXSHUF && (p.ps_s < 1 || p.ps_cout < 2 || p.ps_cout % 2 || p.N != p.ps_s * p.ps_s * p.ps_cout)) {
        set_error("%s: pixel shuffle needs an even channel count and N = s*s*cout (s=%d cout=%d N=%d)", who, p.ps_s, p.ps_cout, p.N);
        return DM_E_INVALID;
    }
    if ((p.epi == EPI_RESID_F32 || p.epi == EPI_HEAD) && !p.gamma) { set_error("%s: gamma is NULL", who); return DM_E_INVALID; }
    if (misaligned(p.bias, 8) || misaligned(p.gamma, 8) || (f32_rows && misaligned(p.X, 8))) { set_error("%s: fp32 operands must be 8-byte aligned", who); return DM_E_INVALID; }
    if (f16_rows && (misaligned(p.C, 4) || misaligned(p.C2, 4) || misaligned(p.R, 4) || misaligned(p.R2, 4))) { set_error("%s: fp16 operands must be 4-byte aligned", who); return DM_E_INVALID; }
    return DM_OK;
}

// N tile of one consumer warpgroup; its M tile is tile_m(bn).  The fused head keeps a whole output row in one tile
// (BN = N = 32).  N % 256 == 0 takes 64 x 256 (m64n256k16: B is read from shared memory once per 256 columns instead of
// twice), the rest 128 x 128, 128 x 64 or 128 x 32.  The two shapes give bit-identical results.  Their speed was compared
// (tools/bench_gemm_micro.py, H100) only on an earlier build whose epilogue overflowed the instruction cache: 64 x 256 was
// up to 7 % faster on qkv, 128 x 128 up to 12 % faster on the decoder's 3x3 convolutions; not re-measured since.
static int pick_bn(const GemmParams &p) {
    if (p.epi == EPI_HEAD) return 32;
    return p.N % 256 == 0 ? 256 : (p.N % 128 == 0 ? 128 : (p.N % 64 == 0 ? 64 : 32));
}
static int tile_m(int bn) { return bn == 256 ? 64 : 128; }

// split mode: the weight-scale vector, and output / residual rows wide enough for their [hi | lo | hi] thirds
static int check_split(const GemmParams &p, const char *who) {
    if (!p.wscale || reinterpret_cast<uintptr_t>(p.wscale) % 8) { set_error("%s: wscale missing or not 8-byte aligned", who); return DM_E_INVALID; }
    const bool f16_out = p.epi == EPI_STORE_F16;
    if ((f16_out && p.ldc < 3 * p.N) || (p.R && p.ldr < 3 * p.N) || (p.R2 && p.ldr2 < 3 * p.N)) {
        set_error("%s: split rows need pitches of at least 3N (N=%d ldc=%d ldr=%d ldr2=%d)", who, p.N, p.ldc, p.ldr, p.ldr2);
        return DM_E_INVALID;
    }
    return DM_OK;
}
static int split_bn(const GemmParams &p) { const int bn = pick_bn(p); return bn > 64 ? 64 : bn; }

// Plain GEMM: A fp16 [M, K] (pitch lda), W fp16 [N, K] (pitch ldw)
int gemm_f16(const __half *A, int lda, const __half *W, int ldw, GemmParams p, cudaStream_t stream) {
    if (p.K % 64 != 0 || p.N % 32 != 0) { set_error("gemm_f16: K must be a multiple of 64 and N of 32 (K=%d N=%d)", p.K, p.N); return DM_E_INVALID; }
    if (p.epi == EPI_HEAD && p.N != 32) { set_error("gemm_f16: the fused head needs N = 32 (N=%d)", p.N); return DM_E_UNSUPPORTED; }
    if (int rc0 = check_epilogue_operands(p, "gemm_f16")) return rc0;
    if ((lda % 8) || (ldw % 8)) { set_error("gemm_f16: row pitches must be multiples of 8 elements"); return DM_E_INVALID; }
    const int bn = pick_bn(p), bm = tile_m(bn);
    const int m_tiles = (p.M + bm - 1) / bm;
    CUtensorMap tmA, tmB;
    int rc = make_tmap_2d(&tmA, A, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)lda, (uint32_t)bm, 64);
    if (rc) return rc;
    rc = make_tmap_2d(&tmB, W, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)ldw, (uint32_t)bn, 64);
    if (rc) return rc;
    switch (bn) {
        case 256: return launch_gemm<64, 256, false>(tmA, tmB, p, m_tiles, stream);
        case 128: return launch_gemm<128, 128, false>(tmA, tmB, p, m_tiles, stream);
        case 64: return launch_gemm<128, 64, false>(tmA, tmB, p, m_tiles, stream);
        case 32: return launch_gemm<128, 32, false>(tmA, tmB, p, m_tiles, stream);
    }
    set_error("gemm_f16: unsupported N tile %d", bn);
    return DM_E_UNSUPPORTED;
}

// Split GEMM: A = split activations [M, K] (K = 3x the logical depth), W = split weights [N, K], p.wscale set
int gemm_split(const __half *A, int lda, const __half *W, int ldw, GemmParams p, cudaStream_t stream) {
    if (p.K % 64 != 0 || p.N % 32 != 0) { set_error("gemm_split: K must be a multiple of 64 and N of 32 (K=%d N=%d)", p.K, p.N); return DM_E_INVALID; }
    if (p.epi == EPI_HEAD && p.N != 32) { set_error("gemm_split: the fused head needs N = 32 (N=%d)", p.N); return DM_E_UNSUPPORTED; }
    if (int rc0 = check_epilogue_operands(p, "gemm_split")) return rc0;
    if (int rc0 = check_split(p, "gemm_split")) return rc0;
    if ((lda % 8) || (ldw % 8)) { set_error("gemm_split: row pitches must be multiples of 8 elements"); return DM_E_INVALID; }
    const int bn = split_bn(p);
    const int m_tiles = (p.M + 127) / 128;
    CUtensorMap tmA, tmB;
    int rc = make_tmap_2d(&tmA, A, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)lda, 128, 64);
    if (rc) return rc;
    rc = make_tmap_2d(&tmB, W, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)ldw, (uint32_t)bn, 64);
    if (rc) return rc;
    return bn == 64 ? launch_gemm<128, 64, false, true>(tmA, tmB, p, m_tiles, stream) : launch_gemm<128, 32, false, true>(tmA, tmB, p, m_tiles, stream);
}

// 3x3 stride-1 convolution, NHWC fp16 activations [B,H,W,Cin], weights fp16 [Cout, 9*Cin] ordered (ky, kx, cin).  halo = 0: pad 1
// with zeros, `src` is the activations; halo = 1: `src` is their [B, H+2, W+2, Cin] copy with the padding already in its border.
// split: the split kernel (Cin is then the stored channel count, 3x the logical one)
static int conv3x3_launch(const __half *src, int halo, int B, int H, int W, int Cin, const __half *Wt, GemmParams p, cudaStream_t stream,
                          bool split = false) {
    const int bn = split ? split_bn(p) : pick_bn(p), bm = tile_m(bn);
    // tile = hbox x wbox pixels = bm rows; choose the wbox in {bm, .., 16, 8} with the least padding waste
    int best_w = bm; double best_eff = -1;
    for (int wb = bm; wb >= 8; wb >>= 1) {
        const int hb = bm / wb;
        const double eff = (double)(W * H) / ((double)((W + wb - 1) / wb * wb) * ((H + hb - 1) / hb * hb));
        if (eff > best_eff + 1e-9) { best_eff = eff; best_w = wb; }
    }
    p.wbox = best_w; p.hbox = bm / best_w;
    p.tiles_x = (W + p.wbox - 1) / p.wbox; p.tiles_y = (H + p.hbox - 1) / p.hbox;
    p.cB = B; p.cH = H; p.cW = W; p.cCin = Cin; p.corg = halo;
    p.M = B * H * W; p.K = 9 * Cin;
    const int m_tiles = B * p.tiles_x * p.tiles_y;
    CUtensorMap tmA, tmB;
    int rc = make_tmap_nhwc(&tmA, src, B, H + 2 * halo, W + 2 * halo, Cin, p.hbox, p.wbox);
    if (rc) return rc;
    rc = make_tmap_2d(&tmB, Wt, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K, (uint32_t)bn, 64);
    if (rc) return rc;
    if (split) return bn == 64 ? launch_gemm<128, 64, true, true>(tmA, tmB, p, m_tiles, stream) : launch_gemm<128, 32, true, true>(tmA, tmB, p, m_tiles, stream);
    switch (bn) {
        case 256: return launch_gemm<64, 256, true>(tmA, tmB, p, m_tiles, stream);
        case 128: return launch_gemm<128, 128, true>(tmA, tmB, p, m_tiles, stream);
        case 64: return launch_gemm<128, 64, true>(tmA, tmB, p, m_tiles, stream);
        case 32: return launch_gemm<128, 32, true>(tmA, tmB, p, m_tiles, stream);
    }
    set_error("conv3x3_f16: unsupported N tile %d", bn);
    return DM_E_UNSUPPORTED;
}

static int check_conv3x3(const GemmParams &p, int Cin, const char *who) {
    if (Cin % 64 != 0 || p.N % 32 != 0) { set_error("%s: Cin must be a multiple of 64 and Cout of 32", who); return DM_E_INVALID; }
    if (p.epi == EPI_HEAD && p.N != 32) { set_error("%s: the fused head needs Cout = 32 (Cout=%d)", who, p.N); return DM_E_UNSUPPORTED; }
    return check_epilogue_operands(p, who);
}

int conv3x3_f16(const __half *act, int B, int H, int W, int Cin, const __half *Wt, GemmParams p, cudaStream_t stream) {
    if (int rc = check_conv3x3(p, Cin, "conv3x3_f16")) return rc;
    return conv3x3_launch(act, 0, B, H, W, Cin, Wt, p, stream);
}

// halo[b, y, x, :] = act[b, (y - 1) mod H, (x - 1) mod W, :] for y < H + 2, x < W + 2: what F.pad(mode='circular') gives a 3x3
// pad-1 convolution.  One thread per 8 channels of a halo pixel; C % 8 == 0.
__global__ void __launch_bounds__(256) conv_halo_circular_kernel(const __half *__restrict__ act, int B, int H, int W, int C, __half *__restrict__ halo) {
    const int c8 = C / 8;
    const long long total = (long long)B * (H + 2) * (W + 2) * c8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        long long r = i / c8;
        const int x = (int)(r % (W + 2));
        r /= W + 2;
        const int y = (int)(r % (H + 2));
        const long long b = r / (H + 2);
        const int sy = wrap_index(y - 1, H), sx = wrap_index(x - 1, W);
        reinterpret_cast<uint4 *>(halo)[i] = __ldg(reinterpret_cast<const uint4 *>(act + ((b * H + sy) * W + sx) * C + c));
    }
}

int conv_halo_circular(const __half *act, int B, int H, int W, int C, __half *halo, cudaStream_t stream) {
    if (!act || !halo || B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8) { set_error("dm_circular_halo_f16: bad arguments (C must be a positive multiple of 8)"); return DM_E_INVALID; }
    if ((reinterpret_cast<uintptr_t>(act) | reinterpret_cast<uintptr_t>(halo)) % 16) { set_error("dm_circular_halo_f16: tensors must be 16-byte aligned"); return DM_E_INVALID; }
    static PerDeviceAttr sms(cudaDevAttrMultiProcessorCount);
    const long long total = (long long)B * (H + 2) * (W + 2) * (C / 8);
    const long long blocks = (total + 255) / 256, cap = 16ll * sms.get();
    conv_halo_circular_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, stream>>>(act, B, H, W, C, halo);
    DM_LAUNCH_CHECK("conv_halo_circular_kernel");
    return DM_OK;
}

// 3x3 stride-1 convolution with circular padding (nn.Conv2d(padding_mode='circular')): the halo copy, then the implicit GEMM on it
int conv3x3_circular_f16(const __half *act, __half *halo, int B, int H, int W, int Cin, const __half *Wt, GemmParams p, cudaStream_t stream) {
    if (int rc = check_conv3x3(p, Cin, "conv3x3_circular")) return rc;
    if (int rc = conv_halo_circular(act, B, H, W, Cin, halo, stream)) return rc;
    return conv3x3_launch(halo, 1, B, H, W, Cin, Wt, p, stream);
}

// Split 3x3 convolution: act = split NHWC [B, H, W, 3 Cin]; Wt = split weights [Cout, 9 * 3 Cin], each tap's columns
// [w_hi | w_hi | w_lo]; halo != NULL: circular padding through the halo copy (B*(H+2)*(W+2)*3*Cin fp16)
int conv3x3_split(const __half *act, __half *halo, int B, int H, int W, int Cin, const __half *Wt, GemmParams p, cudaStream_t stream) {
    if (int rc = check_conv3x3(p, Cin, "conv3x3_split")) return rc;
    if (int rc = check_split(p, "conv3x3_split")) return rc;
    if (!halo) return conv3x3_launch(act, 0, B, H, W, 3 * Cin, Wt, p, stream, true);
    if (int rc = conv_halo_circular(act, B, H, W, 3 * Cin, halo, stream)) return rc;
    return conv3x3_launch(halo, 1, B, H, W, 3 * Cin, Wt, p, stream, true);
}

}  // namespace dm

// ---- C-ABI test / building-block entry points ---------------------------------------------------------------------
extern "C" __attribute__((visibility("default"))) int dm_gemm_f16(const void *A, int lda, const void *W, int ldw, const float *bias, void *C,
                                                               int ldc, int M, int N, int K, int act, int out_f32, void *stream) {
    using namespace dm;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = K; p.act = act; p.bias = bias;
    if (out_f32) { p.epi = EPI_STORE_F32; p.X = (float *)C; p.ldx = ldc; }
    else { p.epi = EPI_STORE_F16; p.C = (__half *)C; p.ldc = ldc; }
    return gemm_f16((const __half *)A, lda, (const __half *)W, ldw, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_conv3x3_f16(const void *act, int B, int H, int W, int Cin, const void *Wt, const float *bias,
                                                                  void *out, int Cout, int relu, void *stream) {
    using namespace dm;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.N = Cout; p.act = relu ? ACT_RELU : ACT_NONE; p.bias = bias; p.epi = EPI_STORE_F16; p.C = (__half *)out; p.ldc = Cout;
    return conv3x3_f16((const __half *)act, B, H, W, Cin, (const __half *)Wt, p, (cudaStream_t)stream);
}

static void desc_to_params(const dm_gemm_desc *d, dm::GemmParams &p) {
    memset(&p, 0, sizeof(p));
    p.M = d->M; p.N = d->N; p.K = d->K; p.epi = d->epi; p.act = d->act; p.bias = d->bias;
    p.C = (__half *)d->C; p.ldc = d->ldc; p.C2 = (__half *)d->C2;
    p.R = (const __half *)d->R; p.ldr = d->ldr; p.R2 = (const __half *)d->R2; p.ldr2 = d->ldr2;
    p.X = d->X; p.ldx = d->ldx; p.gamma = d->gamma; p.head_b2 = d->head_b2;
    p.ps_s = d->ps_s; p.ps_cout = d->ps_cout; p.ps_h = d->ps_h; p.ps_w = d->ps_w;
}

extern "C" __attribute__((visibility("default"))) int dm_gemm_ex(const void *A, int lda, const void *W, int ldw, const dm_gemm_desc *d, void *stream) {
    if (!A || !W || !d) { dm::set_error("dm_gemm_ex: null argument"); return DM_E_INVALID; }
    dm::GemmParams p;
    desc_to_params(d, p);
    return dm::gemm_f16((const __half *)A, lda, (const __half *)W, ldw, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_conv3x3_ex(const void *act, int B, int H, int W, int Cin, const void *Wt, const dm_gemm_desc *d, void *stream) {
    if (!act || !Wt || !d) { dm::set_error("dm_conv3x3_ex: null argument"); return DM_E_INVALID; }
    dm::GemmParams p;
    desc_to_params(d, p);
    return dm::conv3x3_f16((const __half *)act, B, H, W, Cin, (const __half *)Wt, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_circular_halo_f16(const void *act, int B, int H, int W, int C, void *halo, void *stream) {
    return dm::conv_halo_circular((const __half *)act, B, H, W, C, (__half *)halo, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_conv3x3_circular_ex(const void *act, void *halo, int B, int H, int W, int Cin, const void *Wt,
                                                                          const dm_gemm_desc *d, void *stream) {
    if (!act || !halo || !Wt || !d) { dm::set_error("dm_conv3x3_circular_ex: null argument"); return DM_E_INVALID; }
    dm::GemmParams p;
    desc_to_params(d, p);
    return dm::conv3x3_circular_f16((const __half *)act, (__half *)halo, B, H, W, Cin, (const __half *)Wt, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_gemm_split_ex(const void *A, int lda, const void *W, int ldw, const float *wscale,
                                                                    const dm_gemm_desc *d, void *stream) {
    if (!A || !W || !d) { dm::set_error("dm_gemm_split_ex: null argument"); return DM_E_INVALID; }
    dm::GemmParams p;
    desc_to_params(d, p);
    p.wscale = wscale;
    return dm::gemm_split((const __half *)A, lda, (const __half *)W, ldw, p, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int dm_conv3x3_split_ex(const void *act, void *halo, int B, int H, int W, int Cin, const void *Wt,
                                                                       const float *wscale, const dm_gemm_desc *d, void *stream) {
    if (!act || !Wt || !d) { dm::set_error("dm_conv3x3_split_ex: null argument"); return DM_E_INVALID; }
    dm::GemmParams p;
    desc_to_params(d, p);
    p.wscale = wscale;
    return dm::conv3x3_split((const __half *)act, (__half *)halo, B, H, W, Cin, (const __half *)Wt, p, (cudaStream_t)stream);
}
