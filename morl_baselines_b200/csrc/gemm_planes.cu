// gemm_planes.cu -- FP32-accurate dense layers on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Replaces the cuBLAS SIMT sgemm calls behind the reference's nn.Linear layers (common/networks.py:10-48, called from
// multi_policy/envelope/envelope.py:59-77, 300, 420, 429) on the 65,536-row effective batch.  The 1e-5 parity bar rules out
// plain TF32/BF16/FP16, so every fp32 operand is carried as a small number of 16-bit PLANES whose sum reproduces it, and a product
// A.B^T is the sum of the significant plane-by-plane tensor-core MMAs, accumulated in fp32 in the registers of a warpgroup.  Two operand formats:
//
//   MORL_FMT_F16X2  (default of the update path)   s x = h0 + h1: two fp16 planes (11 + 11 significand bits) of the operand scaled
//       by a power of two s (device-resident, per tensor) -- exact to 2^-22 relative; THREE MMAs  A1B0 + A0B1 + A0B0  per product
//       (the dropped A1B1 term is O(2^-22)), 4 bytes per element.  Each fp16 x fp16 product is exact in fp32.  fp16 has 5 exponent
//       bits: |s x| must stay below 65,504 (an overflow becomes Inf/NaN downstream AND raises a device flag, morl_plane_overflow_count),
//       elements below 2^-14 / s lose relative (not absolute) accuracy -- the scales are chosen so that this floor sits >= 2^-26 below
//       the typical magnitude (DESIGN.md section 4.6).
//   MORL_FMT_BF16X3 (wide-range format)            x = x0 + x1 + x2: three bf16 planes (8 + 8 + 8 bits, fp32 exponent range, no scale),
//       exact to 2^-24; SIX MMAs  A2B0 + A0B2 + A1B1 + A1B0 + A0B1 + A0B0, 6 bytes per element.
// Either way the result differs from an fp32 GEMM only at the level of its own accumulation-order noise (tests/test_gemm_gpu.py).
//
// K-major kernel anatomy (persistent, one CTA per SM, 384 threads = three warpgroups; setmaxnreg moves the registers of the producer
// warpgroup to the consumers: 232 per consumer thread, 40 per producer thread, so the 128 accumulators and the epilogue fit without spills):
//   warps 0-7: two consumer warpgroups -- each owns 64 of the tile's 128 rows: waits for a stage, issues NPROD x BK/16
//              wgmma.mma_async (M = 64, N = unit width, K = 16) from the staged boxes and hands the stage back to the producer once the
//              MMAs that read it have completed; the accumulators (N / 2 fp32 registers per thread) then go through the epilogue in place:
//              x 2^-(sA+sB), + bias, ReLU / ReLU-mask, then an fp32 row-major store and/or a re-split into planes (the operand format
//              of the next layer) through TMA stores from two staging tiles per warp used in turn, so intermediate activations never
//              exist in fp32 in HBM;
//   warps 8-11: producer warpgroup, one lane of warp 8 issues TMA -- cp.async.bulk.tensor.3d of a [P planes x 128 rows x BK] A box and
//              P x N/32 [32 rows x BK] B boxes per stage (f16x2: BK = 64, 128-byte swizzle, 2 x 96 KB stages at N = 256; bf16x3: BK = 32,
//              64-byte swizzle, 2 x 72 KB), mbarrier ring; it keeps loading the next tile while the consumers are in their epilogue.
// Operands: A [P][M][K] (K-major), B [P][N_pad][K] (K-major), K % BK == 0, N_pad % 32 == 0, N_pad <= 512.  An output wider than 256
// columns runs as two column units [0, 256) and [256, N_pad) of the same tile, each with the shared-memory plan of N_pad = 256.
// bf16x3 chains of hidden layers (gemm_chain_kernel) run the same pipeline -- carve_kplan, the producer's load_unit, the consumer's consume_unit
// and reload_bias -- on their own schedule of units; f16x2 chains run on gemm_chain_resident_kernel, which keeps a CTA's activation tile in
// shared memory through all layers and streams only the weights.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "gemm_tc.cuh"

namespace morl {

constexpr int kGemmBM = 128;
constexpr int kGemmThreads = 384;  // warps 0-7: two consumer warpgroups (wgmma + epilogue), warps 8-11: producer warpgroup (one lane of warp 8 issues TMA)
// 2 x 128 x 232 + 128 x 40 = 64,512 <= 65,536 registers: a consumer thread holds 128 fp32 accumulators and the epilogue's working set without spilling
constexpr int kGemmConsumerRegs = 232, kGemmProducerRegs = 40;
constexpr int kGemmBoxN = 32;      // B rows per TMA box (one plane): any unit width that is a multiple of 32 is a sequence of them

__device__ unsigned int g_plane_overflow;  // number of kernel launches (approx.) that saw an f16x2 element out of fp16 range


// |scaled value| beyond the largest finite fp16: the planes hold Inf / NaN from here on (they propagate to the loss) and the flag says why
__device__ __forceinline__ void note_overflow(float amax) {
    if (amax > 65504.f) atomicAdd(&g_plane_overflow, 1u);
}

#define MORL_DISPATCH_FMT(F_, ...)                                                         \
    switch (F_) {                                                                          \
        case MORL_FMT_BF16X3: { constexpr int kFmt = MORL_FMT_BF16X3; __VA_ARGS__; } break; \
        case MORL_FMT_F16X2: { constexpr int kFmt = MORL_FMT_F16X2; __VA_ARGS__; } break;   \
        default: break;                                                                    \
    }


struct GemmArgs {
    int M, N, N_pad, K;          // N_pad = B rows covered (multiple of 32, <= 512)
    const float* bias;           // [N] or nullptr
    float* c_f32;                // [M, ldc] or nullptr
    int ldc;
    void* c_planes;              // [P][M][ldp] or nullptr (re-split output: operand of the next layer)
    int ldp;                     // columns of a plane row (>= N, multiple of 32; columns [N, ldp) are written as zero)
    long long plane_stride;      // elements between planes
    const uint32_t* bits_in;     // ReLU-backward mask as BITS [M][relu_bits_words(N_pad)] words (see morl_b200.h "ReLU bit masks"), or nullptr
    uint32_t* bits_out;          // forward: bit = (output > 0) per column, same layout, or nullptr
    int bits_ld;                 // words per row of bits_in / bits_out: relu_bits_words(N_pad) (the epilogue visits every chunk below N_pad)
    int n_stages;                // depth of the TMA ring: as many (A box + B boxes) stages as fit (2 at N_pad = 256, more for narrow outputs)
    uint32_t b_stage;            // bytes of one B stage slot (the B rows of a stage rounded up to 1 KB)
    int relu;
    const float* a_scale;        // device scalars (powers of two) the A / B planes were scaled by; nullptr = 1
    const float* b_scale;
    const float* c_scale;        // scale applied to the output before it is re-split into c_planes; nullptr = 1
    int reverse;                 // walk the row tiles from the last to the first (see morl_gemm_planes_f32: L2 reuse between chained layers)
    unsigned long long* stats;   // diagnostics (MORL_GEMM_STATS=1), else nullptr: [0] consumer wait-on-TMA cycles, [1] consumer loop total,
                                 // [2] producer wait-on-free-stage, [3] epilogue busy
    // LayerNorm / dropout epilogue (EPI == kEpiLn only; appended so that the fields above keep their parameter offsets)
    int ln;                      // LayerNorm over the N output columns of a row
    float ln_eps;
    const float* ln_gamma;       // [N] or nullptr = 1
    const float* ln_beta;        // [N] or nullptr = 0
    const unsigned long long* drop_seed;  // device Philox key, or nullptr = no dropout
    const unsigned int* drop_offset;      // device pass counter (Philox counter word 0)
    unsigned int drop_salt;      // layer salt (counter word 1)
    unsigned int drop_thr;       // keep iff draw >= drop_thr = round(p 2^32)
    float drop_scale;            // float(1 / (1 - p))
    uint32_t* drop_bits;         // keep mask [M][relu_bits_words(N)] in the ReLU-bit layout, or nullptr
};

constexpr int kEpiPlain = 0;     // x k_acc + bias [, ReLU / ReLU mask]
constexpr int kEpiLn = 1;        // relu(LN(dropout(x k_acc + bias))) c_scale

// Philox4x32-10 (Salmon et al., SC'11): four 32-bit draws per (counter, key)
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t (&r)[4]) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    r[0] = c0; r[1] = c1; r[2] = c2; r[3] = c3;
}

__device__ unsigned long long g_gemm_stats[8];

// shared-memory plan of the K-major kernel (host and device agree through these)
template <int FMT>
struct KPlan {
    using F = PlaneFmt<FMT>;
    static constexpr int kStages = F::kStages;                                    // ring depth at N_pad = 256
    static constexpr int kMaxStages = 8;                                          // barrier slots (narrow outputs run a deeper ring)
    static constexpr uint32_t kRowB = F::BK * 2;                                  // bytes per staged row = swizzle span
    static constexpr uint32_t kAStage = F::P * kGemmBM * kRowB;                   // A box bytes
    static constexpr uint32_t kBStage = F::P * 256 * kRowB;                       // B bytes of a stage at N_pad = 256
    static constexpr uint32_t kStageC = F::P * 1024;                              // TMA-store tile: P x 16 rows x 64 B; TWO per consumer warp
    static constexpr uint32_t kOffB = kStages * kAStage;
    static constexpr uint32_t kOffC = kOffB + kStages * kBStage;                  // 1024-aligned (all stage sizes are multiples of 1 KB)
    static constexpr uint32_t kOffBar = kOffC + 8 * 2 * kStageC;
    static constexpr uint32_t kOffBias = kOffBar + 256;
    static constexpr uint32_t kBytes = kOffBias + 1024 + 1024;                    // + alignment slack of the dynamic segment
    static_assert(kBytes <= 227 * 1024, "dynamic shared memory of one CTA on sm_90");
};

// The carve of KPlan in the dynamic shared memory of a K-major kernel (gemm_planes_kernel, gemm_chain_kernel)
struct KSmem {
    uint8_t* a;                  // ring stages of A boxes (KPlan::kAStage each)
    uint8_t* b;                  // ring stages of B rows, b_stage bytes each
    uint32_t b_stage;
    uint8_t* c;                  // TMA-store staging tiles, two per consumer warp
    uint64_t* full;              // ring barriers [kMaxStages]
    uint64_t* empty;             // [kMaxStages], followed by the kernel's own barriers
    float* bias;                 // [256]: the biases of the current unit, indexed by column within the unit
};

template <int FMT>
__device__ __forceinline__ KSmem carve_kplan(uint8_t* smem_raw, uint32_t n_stages, uint32_t b_stage) {
    using L = KPlan<FMT>;
    uint8_t* sm = align_1k(smem_raw);
    KSmem s;
    s.a = sm;
    s.b = sm + n_stages * L::kAStage;  // (n_stages * (A + B) <= kOffC, checked on the host)
    s.b_stage = b_stage;
    s.c = sm + L::kOffC;
    s.full = reinterpret_cast<uint64_t*>(sm + L::kOffBar);
    s.empty = s.full + L::kMaxStages;
    s.bias = reinterpret_cast<float*>(sm + L::kOffBias);
    return s;
}

// Producer of one work unit: per K block, wait for a free stage, then one A box (P planes x 128 rows x BK) and the P x n_cnt / 32 B boxes of
// the unit's columns [n_begin, n_begin + n_cnt).  Returns the cycles spent waiting for free stages if `stats`, else 0.
template <int FMT>
__device__ __forceinline__ long long load_unit(const KSmem& s, Ring& ring, const CUtensorMap* tmA, const CUtensorMap* tmB, int row0, int n_begin, int n_cnt,
                                               int n_kblk, bool stats) {
    using F = PlaneFmt<FMT>;
    using L = KPlan<FMT>;
    const uint32_t b_plane = (uint32_t)n_cnt * L::kRowB;
    long long wait_cycles = 0;
    for (int kb = 0; kb < n_kblk; ++kb) {
        const long long c0 = stats ? clock64() : 0;
        g_mbar_wait(&s.empty[ring.stage], ring.phase ^ 1u);
        if (stats) wait_cycles += clock64() - c0;
        uint64_t* full = &s.full[ring.stage];
        g_mbar_expect_tx(full, L::kAStage + (uint32_t)F::P * b_plane);
        tma_load_3d(s.a + ring.stage * L::kAStage, tmA, full, kb * F::BK, row0, 0);
        uint8_t* bs = s.b + ring.stage * s.b_stage;
        for (int p = 0; p < F::P; ++p)
            for (int r = 0; r < n_cnt; r += kGemmBoxN) tma_load_3d(bs + (uint32_t)p * b_plane + (uint32_t)r * L::kRowB, tmB, full, kb * F::BK, n_begin + r, p);
        ring.advance();
    }
    return wait_cycles;
}

// One work unit of a consumer warpgroup: D[64 x N] = sum over the K blocks of the staged planes, NPROD products per K step in the order of
// PlaneFmt (small terms first).  A stage goes back to the producer as soon as the MMAs reading it have completed: one group of
// wgmma stays in flight while the next stage is awaited.
// SPLIT = 1 ("split accumulators", N <= 128): the tensor cores accumulate in fp32 with limited-precision alignment at every MMA; with all
// NPROD x K/16 products in one accumulator the rounding of the correction products happens at the magnitude of the running sum.  In split
// mode the LEADING products A0B0 go to acc[0, 64) and the correction products (2^-11 / 2^-8 of the magnitude) to acc[64, 128), so only
// K/16 accumulations happen at full magnitude; the epilogue adds the two with one correctly rounded fp32 add.
template <int FMT, int N, int SPLIT>
__device__ __forceinline__ void mma_unit(float (&acc)[128], const KSmem& s, Ring& ring, int n_kblk, int wg, int lane, long long* wait_cycles) {
    using F = PlaneFmt<FMT>;
    static_assert(!SPLIT || N <= 128, "split accumulators: two N / 2-register accumulators per thread");
    constexpr uint32_t ROWB = F::BK * 2;
    constexpr uint32_t a_plane = kGemmBM * ROWB, b_plane = (uint32_t)N * ROWB;
    uint32_t prev = 0;
    for (int kb = 0; kb < n_kblk; ++kb) {
        const long long c0 = wait_cycles ? clock64() : 0;
        g_mbar_wait(&s.full[ring.stage], ring.phase);
        if (wait_cycles) *wait_cycles += clock64() - c0;
        wgmma_fence();
        const uint32_t a0 = g_smem_u32(s.a + ring.stage * KPlan<FMT>::kAStage) + (uint32_t)wg * 64u * ROWB;
        const uint32_t b0 = g_smem_u32(s.b + ring.stage * s.b_stage);
#pragma unroll
        for (int ks = 0; ks < F::BK / 16; ++ks) {
#pragma unroll
            for (int t = 0; t < F::NPROD; ++t) {
                const uint64_t ad = make_desc_k<ROWB>(a0 + F::pa(t) * a_plane + ks * 32);
                const uint64_t bd = make_desc_k<ROWB>(b0 + F::pb(t) * b_plane + ks * 32);
                const bool lead = t == F::NPROD - 1;  // the last product of the list is the leading one (A0B0)
                float* d = (SPLIT && !lead) ? acc + 64 : acc;
                const uint32_t accumulate = SPLIT ? ((lead ? (kb | ks) : (kb | ks | t)) != 0 ? 1u : 0u) : ((kb | ks | t) != 0 ? 1u : 0u);
                Wgmma<N>::template mma<FMT, 0, 0>(d, ad, bd, accumulate);
            }
        }
        wgmma_commit();
        if (kb > 0) {
            wgmma_wait<1>();  // the MMAs of the previous stage have read it
            if (lane == 0) g_mbar_arrive(&s.empty[prev]);
        }
        prev = ring.stage;
        ring.advance();
    }
    wgmma_wait<0>();
    if (n_kblk > 0 && lane == 0) g_mbar_arrive(&s.empty[prev]);
}

struct EpiArgs {
    int M, N;                    // valid rows / columns of the output
    float k_acc;                 // accumulator multiplier (operand scales and folded output scale)
    float c_mul;                 // output scale applied before the re-split when it is not folded into k_acc
    const float* bias_s;         // shared memory, indexed by output column
    int relu;
    const uint32_t* bits_in;
    uint32_t* bits_out;
    int bits_ld;                 // words per bit-mask row (relu_bits_words)
    float* c_f32;
    int ldc;
    int planes;                  // re-split the output into planes through tmC
    int ldp;
};

// Epilogue of one 32-column chunk of a consumer warp's 16 accumulator rows [rbase, rbase + 16): thread l holds a[4 q + 2 h + e] = column
// col0 + 8 q + 2 (l % 4) + e of row rbase + l / 4 + 8 h (the wgmma fragment).  The re-split planes leave through the warp's two staging tiles in
// turn (n_stored counts the warp's bulk stores): a chunk is staged while the TMA store of the previous one is still reading the other tile.
// PRE: a[] already holds the pre-activation (the LayerNorm epilogue has applied scale, bias, dropout and LayerNorm).
// The output values of such a chunk, x[h][2 q + c] = column col0 + 8 q + 2 (l % 4) + c of row rbase + l / 4 + 8 h: scale, bias, ReLU, the
// ReLU-backward bits applied, the ReLU bits recorded.
template <bool PRE>
__device__ __forceinline__ void epilogue_values(const float (&a)[16], int col0, int rbase, int lane, const EpiArgs& e, float (&x)[2][8]) {
    const int l4 = lane & 3, lr = lane >> 2;
    // ReLU bit masks: the word of the row that holds columns [col0, col0 + 32)
    const int wi = relu_bits_word(col0);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                float f;
                if constexpr (PRE) f = a[4 * q + 2 * h + c];
                else f = __fmaf_rn(a[4 * q + 2 * h + c], e.k_acc, e.bias_s[col0 + 8 * q + 2 * l4 + c]);
                if (e.relu) f = (f < 0.f) ? 0.f : f;  // (NaN stays NaN, like torch.relu: an overflow upstream must reach the loss)
                x[h][2 * q + c] = f;
            }
    if (e.bits_in) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rbase + lr + 8 * h;
            const uint32_t keep = row < e.M ? __ldg(e.bits_in + (size_t)row * e.bits_ld + wi) : 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (!((keep >> (8 * (j >> 1) + 2 * l4 + (j & 1))) & 1u)) x[h][j] = 0.f;
        }
    }
    if (e.bits_out) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rbase + lr + 8 * h;
            uint32_t positive = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (x[h][j] > 0.f) positive |= 1u << (8 * (j >> 1) + 2 * l4 + (j & 1));
            positive |= __shfl_xor_sync(0xffffffffu, positive, 1);  // the four threads of a row hold 8 of its 32 columns each
            positive |= __shfl_xor_sync(0xffffffffu, positive, 2);
            if (l4 == 0 && row < e.M) e.bits_out[(size_t)row * e.bits_ld + wi] = positive;
        }
    }
}

// A thread's x[2][8] of such a chunk re-split into P planes of [16 rows][64 B] in shared memory, plane p at base + p plane_stride, in the
// 64-byte swizzle of a TMA box (16-byte chunk q of row r at q ^ ((r >> 1) & 3): bank-conflict free), two columns per word
template <int FMT>
__device__ __forceinline__ void stage_chunk_planes(const float (&x)[2][8], uint8_t* base, uint32_t plane_stride, int lane, float& amax) {
    using F = PlaneFmt<FMT>;
    const int l4 = lane & 3, lr = lane >> 2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int rl = lr + 8 * h;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint32_t w[F::P];
            F::split2(x[h][2 * q], x[h][2 * q + 1], w, amax);
            uint8_t* st = base + rl * 64 + ((q ^ ((rl >> 1) & 3)) << 4) + 4 * l4;
#pragma unroll
            for (int p = 0; p < F::P; ++p) *reinterpret_cast<uint32_t*>(st + p * plane_stride) = w[p];
        }
    }
}

template <int FMT, bool PRE = false>
__device__ __forceinline__ void epilogue_chunk(const float (&a)[16], int col0, int rbase, int lane, const EpiArgs& e, const CUtensorMap* tmC,
                                               uint8_t* my_stage, uint32_t& n_stored, float& amax) {
    constexpr int P = PlaneFmt<FMT>::P;
    const int l4 = lane & 3, lr = lane >> 2;
    float x[2][8];
    epilogue_values<PRE>(a, col0, rbase, lane, e, x);
    if (e.c_f32) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rbase + lr + 8 * h;
            if (row < e.M) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int col = col0 + 8 * q + 2 * l4;
                    float* p = e.c_f32 + (size_t)row * e.ldc + col;
                    if (col + 1 < e.N && (e.ldc & 1) == 0) {
                        *reinterpret_cast<float2*>(p) = make_float2(x[h][2 * q], x[h][2 * q + 1]);
                    } else {
                        if (col < e.N) p[0] = x[h][2 * q];
                        if (col + 1 < e.N) p[1] = x[h][2 * q + 1];
                    }
                }
            }
        }
    }
    if (e.planes && col0 < e.ldp) {
        // stage the warp's [16 rows x 32 cols] x P planes in shared memory, then ONE bulk tensor store writes it out coalesced and asynchronously
        uint8_t* tile = my_stage + (n_stored & 1u) * (uint32_t)(P * 1024);
        ++n_stored;
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // the store before the previous one has read this tile
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int col = col0 + 8 * q + 2 * l4;
                // (c_scale x); ragged last chunk: columns [N, ldp) are written as zero
                x[h][2 * q] = col < e.N ? x[h][2 * q] * e.c_mul : 0.f;
                x[h][2 * q + 1] = col + 1 < e.N ? x[h][2 * q + 1] * e.c_mul : 0.f;
            }
        stage_chunk_planes<FMT>(x, tile, 1024, lane, amax);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
            asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmC), "r"(g_smem_u32(tile)),
                         "r"(col0), "r"(rbase), "r"(0)
                         : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
}

// LayerNorm / dropout epilogue, in place on a consumer warp's accumulators (one column unit holds all N <= 256 columns of its 64 rows;
// thread l holds rows rbase + l / 4 and rbase + l / 4 + 8, acc[16 c + 4 q + 2 h + e] = column 32 c + 8 q + 2 (l % 4) + e of row h):
//   x = acc k_acc + bias;  dropout: x = keep ? x drop_scale : 0 with keep = draw >= drop_thr;  LayerNorm: (x - mean) rstd gamma + beta
// with the two-pass fp32 mean and biased variance of the row (per-thread partial sums + two quad shuffles), rstd = rsqrt(var + eps).
// Draws: Philox4x32-10, key = seed, counter = (*drop_offset, drop_salt, row, g) with column group g = 8 c + 2 (l % 4) + k; draw i of group
// g is column 32 c + 8 (2 k + i / 2) + 2 (l % 4) + i % 2.  Each draw is made once and applied in place, before the statistics.
__device__ __forceinline__ void ln_dropout_unit(float (&acc)[128], int N, int rbase, int lane, const float* bias_s, float k_acc, const GemmArgs& g,
                                                uint32_t k0, uint32_t k1, uint32_t ctr0) {
    const int l4 = lane & 3, lr = lane >> 2;
    const bool drop = g.drop_seed != nullptr;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (32 * c < N) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = rbase + lr + 8 * h;
                uint32_t kept = 0;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    uint32_t r[4] = {0u, 0u, 0u, 0u};
                    if (drop) philox4x32_10(ctr0, g.drop_salt, (uint32_t)row, (uint32_t)(8 * c + 2 * l4 + k), k0, k1, r);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int q = 2 * k + (i >> 1), e = i & 1;
                        const int j = 16 * c + 4 * q + 2 * h + e;
                        float x = __fmaf_rn(acc[j], k_acc, bias_s[32 * c + 8 * q + 2 * l4 + e]);
                        if (drop) {
                            const bool keep = r[i] >= g.drop_thr;
                            x = keep ? __fmul_rn(x, g.drop_scale) : 0.f;
                            kept |= (keep ? 1u : 0u) << (8 * q + 2 * l4 + e);
                        }
                        acc[j] = x;
                    }
                }
                if (g.drop_bits) {
                    kept |= __shfl_xor_sync(0xffffffffu, kept, 1);
                    kept |= __shfl_xor_sync(0xffffffffu, kept, 2);
                    if (l4 == 0 && row < g.M) g.drop_bits[(size_t)row * relu_bits_words(N) + relu_bits_word(32 * c)] = kept;
                }
            }
        }
    }
    if (!g.ln) return;
    const float inv_n = 1.0f / (float)N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (32 * c < N)
#pragma unroll
                for (int t = 0; t < 8; ++t) s = __fadd_rn(s, acc[16 * c + 4 * (t >> 1) + 2 * h + (t & 1)]);
        s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1));
        s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 2));
        const float mean = __fmul_rn(s, inv_n);
        float v = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (32 * c < N)
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    const float d = __fsub_rn(acc[16 * c + 4 * (t >> 1) + 2 * h + (t & 1)], mean);
                    v = __fmaf_rn(d, d, v);
                }
        v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 1));
        v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
        const float rstd = rsqrtf(__fadd_rn(__fmul_rn(v, inv_n), g.ln_eps));
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (32 * c < N)
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    const int col = 32 * c + 8 * (t >> 1) + 2 * l4 + (t & 1);
                    const int j = 16 * c + 4 * (t >> 1) + 2 * h + (t & 1);
                    const float gm = g.ln_gamma ? __ldg(g.ln_gamma + col) : 1.0f, bt = g.ln_beta ? __ldg(g.ln_beta + col) : 0.0f;
                    acc[j] = __fmaf_rn(__fmul_rn(__fsub_rn(acc[j], mean), rstd), gm, bt);
                }
    }
}

// bias_s[c] = mul * bias[n_begin + c] for the 256 columns of a unit (0 at and beyond n_end, or without a bias), by the 256 threads of the
// consumer warps; the first barrier waits until every consumer warp has left the previous unit's epilogue
__device__ __forceinline__ void reload_bias(float* bias_s, const float* bias, int n_begin, int n_end, float mul) {
    bar_sync_named(1, 256);
    const int col = n_begin + (int)threadIdx.x;
    bias_s[threadIdx.x] = (bias && col < n_end) ? __ldg(bias + col) * mul : 0.f;
    bar_sync_named(1, 256);
}

// Consumer warp of one work unit of the columns [n_begin, n_begin + n_cnt): the MMAs of its K blocks (mma_unit at the unit's width), then
// after_mma() (the per-layer kernel: the biases of a wide output's unit, the LayerNorm / dropout pre-pass), then the 32-column chunks of the
// epilogue (split accumulators added first).
template <int FMT, int SPLIT, bool PRE, typename AfterMma>
__device__ __forceinline__ void consume_unit(float (&acc)[128], const KSmem& s, Ring& ring, int n_kblk, int n_begin, int n_cnt, int rbase, int wg, int lane,
                                             long long* wait_cycles, AfterMma&& after_mma, const EpiArgs& e, const CUtensorMap* tmC, uint8_t* my_stage,
                                             uint32_t& n_stored, float& amax) {
#define MORL_UNIT(N_) \
    case N_: mma_unit<FMT, N_, SPLIT>(acc, s, ring, n_kblk, wg, lane, wait_cycles); break;
    switch (n_cnt) {
        MORL_UNIT(32) MORL_UNIT(64) MORL_UNIT(96) MORL_UNIT(128)
        default:
            if constexpr (!SPLIT) {
                switch (n_cnt) {
                    MORL_UNIT(160) MORL_UNIT(192) MORL_UNIT(224) MORL_UNIT(256)
                    default: __trap();
                }
            } else {
                __trap();
            }
    }
#undef MORL_UNIT
    after_mma();
#pragma unroll
    for (int c = 0; c < (SPLIT ? 4 : 8); ++c) {
        if (32 * c < n_cnt) {
            float a[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) a[j] = SPLIT ? __fadd_rn(acc[16 * c + j], acc[64 + 16 * c + j]) : acc[16 * c + j];
            epilogue_chunk<FMT, PRE>(a, n_begin + 32 * c, rbase, lane, e, tmC, my_stage, n_stored, amax);
        }
    }
}

// One CTA per 128-row tile.  SPLIT = 1: see mma_unit; a tile wider than 128 columns is then computed as column units of 128 (the A boxes of
// the tile are staged once per unit).  SPLIT = 0 and N_pad > 256: two column units [0, 256) and [256, N_pad), each with the stage plan of
// N_pad = 256 and this unit's 256 biases in shared memory.  EPI = kEpiLn (SPLIT = 0, N = N_pad <= 256): ln_dropout_unit before the chunks.
template <int FMT, int SPLIT, int EPI = kEpiPlain>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_planes_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                   const GemmArgs g) {
    using L = KPlan<FMT>;
    extern __shared__ uint8_t gsmem_raw[];
    // (ring depth g.n_stages at run time: narrow outputs leave room for a deeper ring, host: morl_gemm_planes_f32)
    const KSmem s = carve_kplan<FMT>(gsmem_raw, (uint32_t)g.n_stages, g.b_stage);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int BN = g.N_pad;
    const int n_tiles = (g.M + kGemmBM - 1) / kGemmBM;
    const int n_kblk = g.K / PlaneFmt<FMT>::BK;
    // Work units: a tile, or its column units of at most kUnitN columns ([0, 128), [128, 256), ... with split accumulators; [0, 256) and
    // [256, BN) for outputs wider than 256 columns).  Both roles enumerate the same sequence.
    constexpr int kUnitN = SPLIT ? 128 : 256;
    const int col_units = (BN + kUnitN - 1) / kUnitN;
    const bool wide = BN > 256;  // the biases of one unit at a time in shared memory (bias_s holds 256)
    const int n_work = n_tiles * col_units;
    auto unit_of = [&](int u, int& tile, int& n_begin, int& n_cnt) {
        tile = u / col_units;
        n_begin = (u - tile * col_units) * kUnitN;
        n_cnt = BN - n_begin < kUnitN ? BN - n_begin : kUnitN;
        if (g.reverse) tile = n_tiles - 1 - tile;
    };

    if (threadIdx.x == 0) {
        init_ring_barriers(s.full, s.empty, (uint32_t)g.n_stages);
        g_mbar_init_fence();
    }
    pdl_enter();  // nothing above reads global memory, everything below may
    for (int t = threadIdx.x; t < 256; t += blockDim.x) s.bias[t] = (g.bias && t < g.N) ? g.bias[t] : 0.f;
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: one lane issues TMA =================
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
            Ring ring((uint32_t)g.n_stages);
            long long w_empty = 0;
            for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
                int tile, n_begin, n_cnt;
                unit_of(u, tile, n_begin, n_cnt);
                w_empty += load_unit<FMT>(s, ring, &tmA, &tmB, tile * kGemmBM, n_begin, n_cnt, n_kblk, g.stats != nullptr);
            }
            if (g.stats) atomicAdd(&g.stats[2], (unsigned long long)w_empty);
        }
    } else {
        // ================= consumer warpgroups (warps 0..7) =================
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2;
        uint8_t* my_stage = s.c + warp * 2 * L::kStageC;
        uint32_t n_stored = 0;
        // x = acc / (sA sB) + bias; when only planes are written (the hidden layers) the output scale is FOLDED into the two constants:
        // fold * x = acc * (fold / (sA sB)) + fold * bias (exact, powers of two), and max / mask commute with a positive factor
        const float c_mul = ld_scale(g.c_scale);
        // (LayerNorm is not scale-invariant through eps: its output scale is applied after the ReLU instead)
        const bool folded = EPI == kEpiPlain && g.c_f32 == nullptr;
        const float fold = folded ? c_mul : 1.0f;
        if (warp == 0 && folded)  // (bias_s was filled before the CTA barrier; one warp rescales it)
            for (int t = lane; t < 256; t += 32) s.bias[t] *= fold;
        bar_sync_named(1, 256);  // the 8 consumer warps only
        EpiArgs e;
        e.M = g.M; e.N = g.N;
        e.k_acc = fold / (ld_scale(g.a_scale) * ld_scale(g.b_scale));
        e.c_mul = folded ? 1.0f : c_mul;
        e.bias_s = s.bias; e.relu = g.relu; e.bits_in = g.bits_in; e.bits_out = g.bits_out; e.bits_ld = g.bits_ld;
        e.c_f32 = g.c_f32; e.ldc = g.ldc; e.planes = g.c_planes != nullptr; e.ldp = g.ldp;
        uint32_t key0 = 0, key1 = 0, ctr0 = 0;
        if constexpr (EPI == kEpiLn) {
            if (g.drop_seed) {
                const unsigned long long seed = *g.drop_seed;
                key0 = (uint32_t)seed;
                key1 = (uint32_t)(seed >> 32);
                ctr0 = *g.drop_offset;
            }
        }
        float amax = 0.f;
        float acc[128];
        Ring ring((uint32_t)g.n_stages);
        long long w_full = 0, busy = 0;
        const long long t_begin = g.stats ? clock64() : 0;
        for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
            int tile, n_begin, n_cnt;
            unit_of(u, tile, n_begin, n_cnt);
            const int rbase = tile * kGemmBM + wg * 64 + (warp & 3) * 16;
            long long c1 = 0;
            consume_unit<FMT, SPLIT, EPI == kEpiLn>(acc, s, ring, n_kblk, n_begin, n_cnt, rbase, wg, lane, g.stats ? &w_full : nullptr, [&] {
                c1 = g.stats ? clock64() : 0;
                if (wide) {
                    // this unit's biases (times the folded output scale), indexed by output column: both warpgroups have finished the MMAs of this unit
                    reload_bias(s.bias, g.bias, n_begin, g.N, fold);
                    e.bias_s = s.bias - n_begin;
                }
                if constexpr (EPI == kEpiLn) ln_dropout_unit(acc, n_cnt, rbase, lane, s.bias, e.k_acc, g, key0, key1, ctr0);
            }, e, &tmC, my_stage, n_stored, amax);
            if (g.stats) busy += clock64() - c1;
        }
        if (g.stats && warp == 0 && lane == 0) {
            atomicAdd(&g.stats[0], (unsigned long long)w_full);
            atomicAdd(&g.stats[1], (unsigned long long)(clock64() - t_begin));
            atomicAdd(&g.stats[3], (unsigned long long)busy);
        }
        if (FMT == MORL_FMT_F16X2) note_overflow(amax);
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all bulk stores of this warp have completed
    }
}

// =================================================================================================================
// CHAIN kernel: several dense hidden layers of one or two networks in ONE persistent launch (bf16x3 planes, N = 256 wide layers; f16x2
// chains run on the resident kernel below).  A layer's output rows depend only on the same rows of its input, so a CTA can take one of
// its 128-row tiles through ALL layers: the tile it stores for layer l is the tile it loads for layer l+1 a few units later -- by then
// still in the 50 MB L2, so only the first layer's input is read from HBM, and the launch prologue / drain is paid once instead of per
// layer.  Work of a CTA: its tiles in groups of `lanes / n_chains`; per group, for every layer, one unit per LANE (lane = (chain, tile
// of the group)): four lanes keep the dependency distance at four units (unit (l, lane) needs the stores of unit (l-1, lane)), so the
// producer never waits for the epilogue that has just finished.  The shared-memory carve, the producer's load_unit and the consumer's
// consume_unit are those of gemm_planes_kernel<bf16x3, 0> (bit-identical outputs: tests/test_gemm_gpu.py); additional barrier stored[lane]:
// the consumer warps arrive once their bulk stores of the unit have COMPLETED, the producer waits for it before loading the next layer of
// that lane.
// =================================================================================================================
constexpr int kChainMaxJobs = 8;   // chains x layers
constexpr int kChainLanes = 4;

// The tiles of both chain kernels on CTA `unit` of n_units: tile t of chain c goes to CTA (t + offset_c) mod n_units with a DIFFERENT rotation
// per chain: when the tiles do not divide evenly, both chains on the same CTAs would give some CTAs two extra tiles and others none; chain 1
// rotated by half the grid spreads the remainders (host model: tests/chain_tiles.py).
struct ChainTiles {
    int cu0, cu1, mt0, mt1, n_units;
    __device__ __forceinline__ ChainTiles(int n_tiles, int n_units_, int n_chains, int unit)
        : cu0(unit), cu1((unit + n_units_ / 2) % n_units_), n_units(n_units_) {
        mt0 = cu0 < n_tiles ? (n_tiles - cu0 + n_units - 1) / n_units : 0;
        mt1 = n_chains > 1 && cu1 < n_tiles ? (n_tiles - cu1 + n_units - 1) / n_units : 0;
    }
    // number of tiles of chain c on this CTA
    __device__ __forceinline__ int count(int c) const { return c ? mt1 : mt0; }
    // first row of tile index ti of chain c on this CTA, or -1
    __device__ __forceinline__ int row(int ti, int c) const { return ti < count(c) ? ((c ? cu1 : cu0) + ti * n_units) * kGemmBM : -1; }
};

struct alignas(64) ChainMaps {
    CUtensorMap A[kChainMaxJobs];  // load map of the INPUT of job (chain c, layer l): [P][M][K], box P x 128 x BK
    CUtensorMap B[kChainMaxJobs];  // weight planes of the job: [P][256][K], box 1 x 32 x BK
    CUtensorMap C[kChainMaxJobs];  // store map of the OUTPUT of the job: [P][M][256], box P x 16 x 32 (64-byte swizzle)
};

// Arguments of both chain kernels (host: set_chain_args); job (c, l) = layer l of chain c, index c n_layers + l
struct ChainArgs {
    int M, K;                      // rows, reduction length (= width of the layers: square 256-wide layers, K % BK == 0)
    int k_first;                   // reduction length of layer 0 of every chain (its INPUT may be narrower: the dX product of the output layer), K % BK == 0
    int n_chains, n_layers;
    const float* bias[kChainMaxJobs];
    const float* b_scale[kChainMaxJobs];
    uint32_t* bits_out[kChainMaxJobs];  // ReLU bit masks of the job's output, or nullptr
    const uint32_t* bits_in[kChainMaxJobs];  // ReLU-backward masks applied to the job's output (dX chains), or nullptr
    const float* a_scale;          // activation scale (input AND output of every layer), device scalar or nullptr
    int relu;                      // max(x, 0) on every job's output (forward chains)
    int n_stages;                  // TMA ring depth of gemm_chain_kernel (KPlan<bf16x3>::kStages; the resident kernel has its own)
};

__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_chain_kernel(const __grid_constant__ ChainMaps maps, const ChainArgs g) {
    constexpr int FMT = MORL_FMT_BF16X3;
    using L = KPlan<FMT>;
    constexpr int BN = 256;
    extern __shared__ uint8_t gsmem_raw[];
    const KSmem s = carve_kplan<FMT>(gsmem_raw, (uint32_t)g.n_stages, L::kBStage);
    uint64_t* stored = s.empty + L::kMaxStages;  // [kChainLanes]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_kblk_full = g.K / PlaneFmt<FMT>::BK, n_kblk_first = g.k_first / PlaneFmt<FMT>::BK;
    const int tiles_per_group = kChainLanes / g.n_chains;  // lanes of a group: (tile of the group) x (chain)
    const ChainTiles tiles((g.M + kGemmBM - 1) / kGemmBM, gridDim.x, g.n_chains, blockIdx.x);
    const int n_groups = (max(tiles.count(0), tiles.count(1)) + tiles_per_group - 1) / tiles_per_group;
    // unit (group gi, layer l, lane ln) -> (job, first row of its tile) or row0 = -1 (no such tile for this CTA)
    auto unit_of = [&](int gi, int l, int ln, int& job, int& row0) {
        const int c = ln % g.n_chains;
        job = c * g.n_layers + l;
        row0 = tiles.row(gi * tiles_per_group + ln / g.n_chains, c);
    };

    if (threadIdx.x == 0) {
        init_ring_barriers(s.full, s.empty, (uint32_t)g.n_stages);
        for (int i = 0; i < kChainLanes; ++i) g_mbar_init(&stored[i], 8);  // the 8 consumer warps
        g_mbar_init_fence();
    }
    pdl_enter();
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: one lane issues TMA =================
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            Ring ring((uint32_t)g.n_stages);
            uint32_t done_on_lane[kChainLanes] = {0u, 0u, 0u, 0u};  // units already issued on each lane = completions of stored[lane] to expect
            for (int gi = 0; gi < n_groups; ++gi)
                for (int l = 0; l < g.n_layers; ++l)
                    for (int ln = 0; ln < kChainLanes; ++ln) {
                        int job, row0;
                        unit_of(gi, l, ln, job, row0);
                        if (row0 < 0) continue;
                        if (l > 0) {
                            // the input tile of this unit is the output tile of the lane's previous unit: wait until the stores of
                            // it have completed (completion number done_on_lane[ln] of stored[ln])
                            g_mbar_wait(&stored[ln], (done_on_lane[ln] - 1u) & 1u);
                            asm volatile("fence.proxy.async.global;" ::: "memory");
                        }
                        ++done_on_lane[ln];
                        load_unit<FMT>(s, ring, &maps.A[job], &maps.B[job], row0, 0, BN, l == 0 ? n_kblk_first : n_kblk_full, false);
                    }
        }
    } else {
        // ================= consumer warpgroups (warps 0..7) =================
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2;
        uint8_t* my_stage = s.c + warp * 2 * L::kStageC;
        uint32_t n_stored = 0;
        const float s_act = ld_scale(g.a_scale);
        float amax = 0.f;
        float acc[128];
        Ring ring((uint32_t)g.n_stages);
        for (int gi = 0; gi < n_groups; ++gi)
            for (int l = 0; l < g.n_layers; ++l)
                for (int ln = 0; ln < kChainLanes; ++ln) {
                    int job, row0;
                    unit_of(gi, l, ln, job, row0);
                    if (row0 < 0) continue;
                    reload_bias(s.bias, g.bias[job], 0, BN, s_act);  // (times the folded output scale)
                    EpiArgs e;
                    e.M = g.M; e.N = BN;
                    // x * s_act = acc * (s_act / (s_act * sB)) + s_act * bias  (powers of two: exact), as gemm_planes_kernel's folded epilogue
                    e.k_acc = s_act / (s_act * ld_scale(g.b_scale[job]));
                    e.c_mul = 1.0f;
                    e.bias_s = s.bias; e.relu = g.relu; e.bits_in = g.bits_in[job]; e.bits_out = g.bits_out[job]; e.bits_ld = relu_bits_words(BN);
                    e.c_f32 = nullptr; e.ldc = 0; e.planes = 1; e.ldp = BN;
                    const int rbase = row0 + wg * 64 + (warp & 3) * 16;
                    consume_unit<FMT, 0, false>(acc, s, ring, l == 0 ? n_kblk_first : n_kblk_full, 0, BN, rbase, wg, lane, nullptr, [] {}, e,
                                                &maps.C[job], my_stage, n_stored, amax);
                    // the lane's next layer loads what this unit stored (bit masks included): signal once the bulk stores of this warp have completed
                    __syncwarp();
                    if (lane == 0) {
                        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
                        g_mbar_arrive(&stored[ln]);
                    }
                }
    }
}

// =================================================================================================================
// RESIDENT chain kernel (f16x2): a CTA keeps its 128-row activation tile in shared memory from the first layer of a chain to the last.
// Layer l's epilogue writes its output chunk c (32 columns) as K-block c of layer l+1's A operand, so no intermediate activation goes
// through L2 and layer l+1 waits for no global store; the producer streams only weights.  An output leaves by TMA store straight from the
// tile only when the job's `store` bit is set.  The chain's input is either a TMA load of plane rows (dX chains, GemmChain) or, in pair mode,
// relu(u[b] + v[j]) s for row b W + j computed by the consumer warps into the tile (pair_split8, as pairs_relu_split_h256_kernel).
// Schedule of a CTA: its tiles in order, each through every layer of chain 0, then (same tile index, the chain's own rotation) chain 1.
// Accumulation order = per-layer gemm_planes_kernel<f16x2, 0> launches': k16 steps in order, products A1B0, A0B1, A0B0 inner (a 32-wide
// K block issues the same sequence as a 64-wide one), so outputs are bit-identical.
// =================================================================================================================
struct ResPlan {
    static constexpr int P = 2, BK = 32, kStages = 3;
    static constexpr uint32_t kRowB = BK * 2;                          // 64 B rows, 64-byte swizzle (make_desc_k<64>)
    static constexpr uint32_t kKBlock = P * kGemmBM * kRowB;           // one K-block of the activation tile: [P][128 rows][64 B] = 16 KB
    static constexpr uint32_t kPlaneKB = kGemmBM * kRowB;              // 8 KB: one plane of a K-block
    static constexpr uint32_t kAct = 8 * kKBlock;                      // 256 columns: 128 KB
    static constexpr uint32_t kBStage = P * 256 * kRowB;               // weights of one K-block: 32 KB
    static constexpr uint32_t kOffB = kAct;
    static constexpr uint32_t kOffBias = kOffB + kStages * kBStage;
    static constexpr uint32_t kOffBar = kOffBias + 1024;
    static constexpr uint32_t kBytes = kOffBar + 256 + 1024;           // + alignment slack of the dynamic segment
    static_assert(kBytes <= 232448, "dynamic shared memory of one CTA on sm_90 (227 KB)");
};

struct alignas(64) ResChainMaps {
    CUtensorMap A[2];              // planes mode: the chain's input [P][M][k_first], box P x 128 x 32
    CUtensorMap B[kChainMaxJobs];  // weight planes of the job [P][256][K], box 1 x 256 x 32
    CUtensorMap C[kChainMaxJobs];  // stored output of the job [P][M][256], box 1 x 16 x 32 (64-byte swizzle)
};

struct ResChainArgs : ChainArgs {
    uint32_t store;                // bit job: the job's output is written to global memory
    const float* u[2];             // pair mode (u != nullptr): u[c] [B][256], v[c] [W][256], row r = b W + j
    const float* v[2];
    int W;
    unsigned long long* stats;     // MORL_GEMM_STATS=1: [0] consumer wait on weights, [1] consumer loop, [2] producer wait on free stage,
                                   // [3] epilogue busy, [4] consumer wait on the input tile (tile boundary)
};

// Consumer warpgroup of one layer: A = its 64 rows of the resident tile, B = the ring.  Same products in the same order as mma_unit.
__device__ __forceinline__ void mma_unit_resident(float (&acc)[128], uint32_t act, const KSmem& s, Ring& ring, int n_kblk, int wg, int lane,
                                                  long long* wait_cycles) {
    using F = PlaneFmt<MORL_FMT_F16X2>;
    using R = ResPlan;
    constexpr uint32_t b_plane = 256u * R::kRowB;
    const uint32_t a_wg = act + (uint32_t)wg * 64u * R::kRowB;
    uint32_t prev = 0;
    for (int kb = 0; kb < n_kblk; ++kb) {
        const long long c0 = wait_cycles ? clock64() : 0;
        g_mbar_wait(&s.full[ring.stage], ring.phase);
        if (wait_cycles) *wait_cycles += clock64() - c0;
        wgmma_fence();
        const uint32_t a0 = a_wg + (uint32_t)kb * R::kKBlock;
        const uint32_t b0 = g_smem_u32(s.b + ring.stage * R::kBStage);
#pragma unroll
        for (int ks = 0; ks < R::BK / 16; ++ks) {
#pragma unroll
            for (int t = 0; t < F::NPROD; ++t) {
                const uint64_t ad = make_desc_k<R::kRowB>(a0 + F::pa(t) * R::kPlaneKB + ks * 32);
                const uint64_t bd = make_desc_k<R::kRowB>(b0 + F::pb(t) * b_plane + ks * 32);
                Wgmma<256>::template mma<MORL_FMT_F16X2, 0, 0>(acc, ad, bd, (kb | ks | t) != 0 ? 1u : 0u);
            }
        }
        wgmma_commit();
        if (kb > 0) {
            wgmma_wait<1>();
            if (lane == 0) g_mbar_arrive(&s.empty[prev]);
        }
        prev = ring.stage;
        ring.advance();
    }
    wgmma_wait<0>();
    if (n_kblk > 0 && lane == 0) g_mbar_arrive(&s.empty[prev]);
}

// 16-byte chunk (8 columns, 4 words per plane) of row `row` (of the tile) in K-block kb of the resident tile (64-byte swizzle)
__device__ __forceinline__ uint8_t* res_chunk(uint8_t* act, int kb, int row, int q) {
    return act + (uint32_t)kb * ResPlan::kKBlock + (uint32_t)row * ResPlan::kRowB + (uint32_t)((q ^ ((row >> 1) & 3)) << 4);
}

// The pair input of 8 consecutive columns from their pre-activations x (u + v, or the product u v): r = relu(x) (NaN-propagating, like
// torch.relu) when `relu`, else r = x; o[p][t] = plane p of (r[2 t] s, r[2 t + 1] s).  Returns bit t = (r[t] > 0).
template <int FMT>
__device__ __forceinline__ uint32_t pair_split8(const float (&x)[8], bool relu, float s, uint32_t (&o)[PlaneFmt<FMT>::P][4], float& amax) {
    using F = PlaneFmt<FMT>;
    uint32_t pos = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        float r0 = x[2 * t], r1 = x[2 * t + 1];
        if (relu) {
            r0 = r0 < 0.f ? 0.f : r0;
            r1 = r1 < 0.f ? 0.f : r1;
        }
        pos |= (r0 > 0.f ? 1u : 0u) << (2 * t) | (r1 > 0.f ? 1u : 0u) << (2 * t + 1);
        uint32_t w[F::P];
        F::split2(r0 * s, r1 * s, w, amax);
#pragma unroll
        for (int p = 0; p < F::P; ++p) o[p][t] = w[p];
    }
    return pos;
}

__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_chain_resident_kernel(const __grid_constant__ ResChainMaps maps, const ResChainArgs g) {
    using R = ResPlan;
    constexpr int P = R::P, BN = 256;
    extern __shared__ uint8_t gsmem_raw[];
    uint8_t* sm = align_1k(gsmem_raw);
    uint8_t* act = sm;
    KSmem s;
    s.a = nullptr;
    s.b = sm + R::kOffB;
    s.b_stage = R::kBStage;
    s.c = nullptr;
    s.bias = reinterpret_cast<float*>(sm + R::kOffBias);
    s.full = reinterpret_cast<uint64_t*>(sm + R::kOffBar);
    s.empty = s.full + R::kStages;
    uint64_t* act_full = s.empty + R::kStages;  // planes mode: the input tile has landed (TMA transaction bytes)
    uint64_t* act_empty = act_full + 1;         // planes mode: the 8 consumer warps are done with the tile (MMAs and stores read it)
    const bool pairs = g.u[0] != nullptr;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_kblk_full = g.K / R::BK, n_kblk_first = g.k_first / R::BK;
    const ChainTiles tiles((g.M + kGemmBM - 1) / kGemmBM, gridDim.x, g.n_chains, blockIdx.x);
    const int n_ti = max(tiles.count(0), tiles.count(1));

    if (threadIdx.x == 0) {
        init_ring_barriers(s.full, s.empty, R::kStages);
        g_mbar_init(act_full, 1);
        g_mbar_init(act_empty, 8);
        g_mbar_init_fence();
    }
    pdl_enter();
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: one lane issues TMA (weights; the input tile in planes mode) =================
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            Ring ring((uint32_t)R::kStages);
            long long w_empty = 0;
            uint32_t n_in = 0;  // input tiles loaded
            for (int ti = 0; ti < n_ti; ++ti)
                for (int c = 0; c < g.n_chains; ++c) {
                    const int row0 = tiles.row(ti, c);
                    if (row0 < 0) continue;
                    for (int l = 0; l < g.n_layers; ++l) {
                        const int job = c * g.n_layers + l;
                        const int nkb = l == 0 ? n_kblk_first : n_kblk_full;
                        for (int kb = 0; kb < nkb; ++kb) {
                            if (!pairs && l == 0 && kb == (nkb < R::kStages ? nkb - 1 : R::kStages - 1)) {
                                // the input tile, once the first weight stages are on their way (they only needed free ring slots): wait
                                // until the consumers are done with the previous tile, then load the k_first / 32 K-blocks of this one
                                if (n_in > 0) {
                                    const long long c0 = g.stats ? clock64() : 0;
                                    g_mbar_wait(act_empty, (n_in - 1u) & 1u);
                                    if (g.stats) w_empty += clock64() - c0;
                                }
                                g_mbar_expect_tx(act_full, (uint32_t)n_kblk_first * R::kKBlock);
                                for (int k = 0; k < n_kblk_first; ++k) tma_load_3d(act + k * R::kKBlock, &maps.A[c], act_full, k * R::BK, row0, 0);
                                ++n_in;
                            }
                            const long long c0 = g.stats ? clock64() : 0;
                            g_mbar_wait(&s.empty[ring.stage], ring.phase ^ 1u);
                            if (g.stats) w_empty += clock64() - c0;
                            uint64_t* full = &s.full[ring.stage];
                            g_mbar_expect_tx(full, R::kBStage);
                            uint8_t* bs = s.b + ring.stage * R::kBStage;
                            for (int p = 0; p < P; ++p) tma_load_3d(bs + (uint32_t)p * 256u * R::kRowB, &maps.B[job], full, kb * R::BK, 0, p);
                            ring.advance();
                        }
                    }
                }
            if (g.stats) atomicAdd(&g.stats[2], (unsigned long long)w_empty);
        }
    } else {
        // ================= consumer warpgroups (warps 0..7) =================
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2, wr = warp & 3;
        const int l4 = lane & 3, lr = lane >> 2;
        const int trow = wg * 64 + wr * 16;  // this warp's 16 rows of the tile
        const float s_act = ld_scale(g.a_scale);
        const uint32_t act_s = g_smem_u32(act);
        float amax = 0.f;
        float acc[128];
        Ring ring((uint32_t)R::kStages);
        long long w_full = 0, busy = 0, w_act = 0;
        const long long t_begin = g.stats ? clock64() : 0;
        uint32_t n_in = 0;
        for (int ti = 0; ti < n_ti; ++ti)
            for (int c = 0; c < g.n_chains; ++c) {
                const int row0 = tiles.row(ti, c);
                if (row0 < 0) continue;
                if (pairs) {
                    // the input tile: relu(u[b] + v[j]) s split into planes, this warp's 16 rows; lane = (row l / 4 + 8 h, 8 columns l % 4 of
                    // every K-block).  The stores of the previous tile's last layer must have read these rows.
                    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    __syncwarp();
                    const float* u = c ? g.u[1] : g.u[0];
                    const float* v = c ? g.v[1] : g.v[0];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int rl = trow + lr + 8 * h, row = row0 + rl;
                        const bool ok = row < g.M;
                        const int b = ok ? row / g.W : 0, j = ok ? row - b * g.W : 0;
#pragma unroll 2
                        for (int kb = 0; kb < 8; ++kb) {
                            const int col = kb * 32 + 8 * l4;
                            uint32_t o[P][4];
                            if (ok) {
                                const float4* up = reinterpret_cast<const float4*>(u + (size_t)b * BN + col);
                                const float4* vp = reinterpret_cast<const float4*>(v + (size_t)j * BN + col);
                                const float4 u0 = __ldg(up), u1 = __ldg(up + 1), v0 = __ldg(vp), v1 = __ldg(vp + 1);
                                const float x[8] = {u0.x + v0.x, u0.y + v0.y, u0.z + v0.z, u0.w + v0.w, u1.x + v1.x, u1.y + v1.y, u1.z + v1.z, u1.w + v1.w};
                                pair_split8<MORL_FMT_F16X2>(x, true, s_act, o, amax);
                            } else {
#pragma unroll
                                for (int t = 0; t < 4; ++t)
#pragma unroll
                                    for (int p = 0; p < P; ++p) o[p][t] = 0u;
                            }
                            uint8_t* dst = res_chunk(act, kb, rl, l4);
#pragma unroll
                            for (int p = 0; p < P; ++p) *reinterpret_cast<uint4*>(dst + p * R::kPlaneKB) = make_uint4(o[p][0], o[p][1], o[p][2], o[p][3]);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    bar_sync_named(2 + wg, 128);  // the warpgroup's 64 rows are in place before its first MMA
                }
                for (int l = 0; l < g.n_layers; ++l) {
                    const int job = c * g.n_layers + l;
                    const bool last = l == g.n_layers - 1, store = (g.store >> job) & 1u;
                    reload_bias(s.bias, g.bias[job], 0, BN, s_act);  // (times the folded output scale; both warpgroups left the previous epilogue)
                    if (!pairs && l == 0) {
                        const long long c0 = g.stats ? clock64() : 0;
                        g_mbar_wait(act_full, n_in & 1u);
                        if (g.stats) w_act += clock64() - c0;
                    }
                    mma_unit_resident(acc, act_s, s, ring, l == 0 ? n_kblk_first : n_kblk_full, wg, lane, g.stats ? &w_full : nullptr);
                    const long long c1 = g.stats ? clock64() : 0;
                    EpiArgs e;
                    e.M = g.M; e.N = BN;
                    e.k_acc = s_act / (s_act * ld_scale(g.b_scale[job]));  // as gemm_planes_kernel's folded epilogue
                    e.c_mul = 1.0f;
                    e.bias_s = s.bias; e.relu = g.relu; e.bits_in = g.bits_in[job]; e.bits_out = g.bits_out[job]; e.bits_ld = relu_bits_words(BN);
                    e.c_f32 = nullptr; e.ldc = 0; e.planes = 1; e.ldp = BN;
                    const bool to_tile = !last || store;
                    if (to_tile) {
                        // the rows are overwritten: the stores of the previous layer (if any) must have read them
                        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                        __syncwarp();
                    }
                    const int rbase = row0 + trow;
#pragma unroll
                    for (int cc = 0; cc < 8; ++cc) {
                        float a[16];
#pragma unroll
                        for (int jj = 0; jj < 16; ++jj) a[jj] = acc[16 * cc + jj];
                        float x[2][8];
                        epilogue_values<false>(a, 32 * cc, rbase, lane, e, x);
                        if (to_tile) {
                            // output chunk cc = K-block cc of the next layer, the swizzled layout of a TMA box [P][128][32] (trow % 16 == 0: the
                            // swizzle of the warp's rows is that of a 16-row staging tile)
                            stage_chunk_planes<MORL_FMT_F16X2>(x, act + cc * R::kKBlock + trow * R::kRowB, R::kPlaneKB, lane, amax);
                            if (store) {
                                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                                __syncwarp();
                                if (lane == 0) {
                                    const uint32_t src = act_s + (uint32_t)cc * R::kKBlock + (uint32_t)trow * R::kRowB;
#pragma unroll
                                    for (int p = 0; p < P; ++p)
                                        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(&maps.C[job]),
                                                     "r"(src + p * R::kPlaneKB), "r"(32 * cc), "r"(rbase), "r"(p)
                                                     : "memory");
                                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                                }
                            }
                        }
                    }
                    if (!last) {
                        // next layer: its A operand (this warpgroup's 64 rows) is complete and visible to the tensor cores
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        bar_sync_named(2 + wg, 128);
                    } else if (!pairs) {
                        // the producer may load the next input tile once every warp's stores have read its rows
                        __syncwarp();
                        if (lane == 0) {
                            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                            g_mbar_arrive(act_empty);
                        }
                    }
                    if (g.stats) busy += clock64() - c1;
                }
                ++n_in;
            }
        if (g.stats && warp == 0 && lane == 0) {
            atomicAdd(&g.stats[0], (unsigned long long)w_full);
            atomicAdd(&g.stats[1], (unsigned long long)(clock64() - t_begin));
            atomicAdd(&g.stats[3], (unsigned long long)busy);
            atomicAdd(&g.stats[4], (unsigned long long)w_act);
        }
        note_overflow(amax);
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all bulk stores of this warp have completed
    }
}

// =================================================================================================================
// MN-major split-K variant: weight gradients  dW[n, k] = sum_m G[m, n] * H[m, k]  (reduction over the 65,536 batch rows).
// Both operands are the row-major plane tensors the forward/backward GEMMs already produced, read "MN-major" (the MMA's M / N
// index is the contiguous one), 128-byte swizzle:  A = G^T (M_mma = n, 128 per CTA: 64 per warpgroup), B = H^T (N_mma = k <= 256), K_mma = m.
// One CTA per (128-row block of n, unit of <= 256 columns of k, split s of the m range); H wider than 256 columns is two k units [0, 256) and
// [256, NB), and only the CTAs of k unit 0 evaluate the fused column sums.  fp32 partial tiles are summed by reduce_partials_kernel
// (deterministic, no atomics), which also removes the operand scales.
// =================================================================================================================
constexpr int kMnKT = 32;  // batch rows (K_mma direction) per pipeline stage

// canonical MN-major layout, SWIZZLE_128B: 64 contiguous MN elements (128 B) x 8 K-rows per 1 KB atom;
// SBO = 1024 B (next 8 K-rows), LBO = distance between 64-element MN chunks.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;  // SWIZZLE_128B
    return d;
}

struct GemmMnArgs {
    int M;            // reduction length (batch rows)
    int n_tiles;      // ceil(A columns / 128)
    int NB;           // B columns covered (multiple of 64, <= 512): N_mma of one k unit (<= 256), or of two ([0, 256) and [256, NB))
    int rows_per_split;
    float* partial;   // [S][n_tiles*128][NB]
    float* colsum_partial;  // [S][n_tiles*128] or nullptr: per-split column sums of G (bias gradient), fused as G^T . ones
};

// One consumer warpgroup of the weight-gradient kernel: acc[64 x NB] = G_chunk^T . H over the stages (cs[64 x 16] = G_chunk^T . ones), then the
// fp32 partial tile of this split.  NB and COLSUM are template parameters and the accumulators live in this function only: a run-time
// branch between the wgmma of one commit group, or one 128-register accumulator array shared by the instantiations of all widths, makes
// ptxas serialise the wgmma (its remarks C7519 / C7511).
template <int FMT, int NB, bool COLSUM>
__device__ __forceinline__ void mma_mn_unit(const GemmMnArgs& g, int split, int row, int col0, uint8_t* smA, uint8_t* smB, uint32_t a_stage, uint32_t b_stage,
                                            uint32_t chunk_bytes, uint64_t ones_desc, int n_kblk, uint64_t* full, uint64_t* empty, int wg, int lane) {
    using F = PlaneFmt<FMT>;
    constexpr int P = F::P;
    constexpr uint32_t plane = kMnKT * 128u;  // 4 KB: one plane of one chunk
    float acc[NB / 2], cs[8];
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;  // (a split without rows writes zeros)
#pragma unroll
    for (int i = 0; i < 8; ++i) cs[i] = 0.f;
    uint32_t stage = 0, phase = 0, prev = 0;
    for (int kb = 0; kb < n_kblk; ++kb) {
        g_mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a0 = g_smem_u32(smA + stage * a_stage) + (uint32_t)wg * chunk_bytes;  // this warpgroup's 64 columns of G
        const uint32_t b0 = g_smem_u32(smB + stage * b_stage);
#pragma unroll
        for (int ks = 0; ks < kMnKT / 16; ++ks) {
#pragma unroll
            for (int t = 0; t < F::NPROD; ++t) {
                const uint64_t ad = make_desc_mn_sw128(a0 + F::pa(t) * plane + ks * 2048u, chunk_bytes);
                const uint64_t bd = make_desc_mn_sw128(b0 + F::pb(t) * plane + ks * 2048u, chunk_bytes);
                Wgmma<NB>::template mma<FMT, 1, 1>(acc, ad, bd, (kb | ks | t) != 0 ? 1u : 0u);
            }
            if constexpr (COLSUM) {  // (G_{P-1} + ... + G_0)^T . ones -> 16 identical columns
#pragma unroll
                for (int pl = P - 1; pl >= 0; --pl)
                    Wgmma<16>::template mma<FMT, 1, 1>(cs, make_desc_mn_sw128(a0 + pl * plane + ks * 2048u, chunk_bytes), ones_desc,
                                                       (kb | ks | (P - 1 - pl)) != 0 ? 1u : 0u);
            }
        }
        wgmma_commit();
        if (kb > 0) {
            wgmma_wait<1>();
            if (lane == 0) g_mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == (uint32_t)F::kStagesMn) {
            stage = 0;
            phase ^= 1u;
        }
    }
    wgmma_wait<0>();
    const int l4 = lane & 3;  // this thread holds output rows (n) row and row + 8
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* prow = g.partial + ((size_t)split * g.n_tiles * 128 + row + 8 * h) * g.NB + col0 + 2 * l4;
#pragma unroll
        for (int j = 0; j < NB / 8; ++j) *reinterpret_cast<float2*>(prow + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        if (COLSUM && l4 == 0) g.colsum_partial[(size_t)split * g.n_tiles * 128 + row + 8 * h] = cs[2 * h];
    }
}

template <int FMT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_planes_mn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmMnArgs g) {
    using F = PlaneFmt<FMT>;
    constexpr int P = F::P;
    constexpr int kStages = F::kStagesMn;
    extern __shared__ uint8_t gsmem_raw[];
    uint8_t* gsmem = align_1k(gsmem_raw);
    constexpr uint32_t chunk_bytes = (uint32_t)P * kMnKT * 128u;   // one 64-element MN chunk, P planes
    constexpr uint32_t a_stage = 2u * chunk_bytes;
    constexpr uint32_t b_stage = 4u * chunk_bytes;                 // (allocated for a k unit of 256 columns)
    const int k_units = g.NB > 256 ? 2 : 1;
    const int col0 = (int)(blockIdx.x / g.n_tiles % k_units) * 256;  // first column of H (k) of this CTA's unit
    const int nb = g.NB - col0 < 256 ? g.NB - col0 : 256;
    const int nb_chunks = nb / 64;
    uint8_t* smA = gsmem;
    uint8_t* smB = gsmem + kStages * a_stage;
    uint64_t* full = reinterpret_cast<uint64_t*>(smB + kStages * b_stage);
    uint64_t* empty = full + kStages;
    // 4 KB of 1.0: the B operand of the fused bias-gradient product  colsum(G) = G^T . ones  (N = 16; every element is 1,
    // so the swizzle pattern is irrelevant)
    uint8_t* ones_b = reinterpret_cast<uint8_t*>(empty + kStages);
    uint32_t* ones = reinterpret_cast<uint32_t*>(align_1k(ones_b));
    for (int t = threadIdx.x; t < 1024; t += blockDim.x) ones[t] = F::kOnes2;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nt = blockIdx.x % g.n_tiles;
    const int split = blockIdx.x / (g.n_tiles * k_units);
    const int m_begin = split * g.rows_per_split;
    const int m_end = min(g.M, m_begin + g.rows_per_split);
    const int n_kblk = (m_end - m_begin + kMnKT - 1) / kMnKT;

    if (threadIdx.x == 0) {
        init_ring_barriers(full, empty, kStages);
        g_mbar_init_fence();
    }
    __syncthreads();
    pdl_enter();  // (nothing above reads or writes global memory: barriers and the tile of ones overlap the predecessor)

    if (warp >= 8) {
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (int kb = 0; kb < n_kblk; ++kb) {
                g_mbar_wait(&empty[stage], phase ^ 1u);
                g_mbar_expect_tx(&full[stage], (2u + (uint32_t)nb_chunks) * chunk_bytes);
                const int m0 = m_begin + kb * kMnKT;
                for (int c = 0; c < 2; ++c) tma_load_3d(smA + stage * a_stage + c * chunk_bytes, &tmA, &full[stage], nt * 128 + c * 64, m0, 0);
                for (int c = 0; c < nb_chunks; ++c) tma_load_3d(smB + stage * b_stage + c * chunk_bytes, &tmB, &full[stage], col0 + c * 64, m0, 0);
                if (++stage == kStages) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
        }
    } else {
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2;
        const uint64_t ones_desc = make_desc_mn_sw128(g_smem_u32(ones), chunk_bytes);
        const bool colsum = g.colsum_partial != nullptr && col0 == 0;
        const int row = nt * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#define MORL_UNIT(N_)                                                                                                                               \
    case N_:                                                                                                                                        \
        if (colsum) mma_mn_unit<FMT, N_, true>(g, split, row, col0, smA, smB, a_stage, b_stage, chunk_bytes, ones_desc, n_kblk, full, empty, wg, lane); \
        else mma_mn_unit<FMT, N_, false>(g, split, row, col0, smA, smB, a_stage, b_stage, chunk_bytes, ones_desc, n_kblk, full, empty, wg, lane);       \
        break;
        switch (nb) {
            MORL_UNIT(64) MORL_UNIT(128) MORL_UNIT(192) MORL_UNIT(256)
            default: __trap();
        }
#undef MORL_UNIT
    }
}

// out[r][c] (or out[c][r] if transpose) = mul * sum_s partial[s][r][c] for r < rows, c < cols, mul = 1 / (scale_a * scale_b).
// blockDim = (32, 8): 32 consecutive output elements per block, the S partials are strided over threadIdx.y (fixed order:
// deterministic), then combined through shared memory.
// Blocks beyond the matrix (blockIdx.x >= main_blocks) reduce the fused column-sum partials vec_partial[s][prow] into vec_out[rows]
// (mul = 1 / scale_a).
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ partial, int S, int prow, int pcol, int rows, int cols,
                                                              int transpose, float* __restrict__ out, int ld_out, int main_blocks,
                                                              const float* __restrict__ vec_partial, float* __restrict__ vec_out,
                                                              const float* __restrict__ scale_a, const float* __restrict__ scale_b) {
    pdl_enter();
    __shared__ float red[8][33];
    float mul = 1.0f / (ld_scale(scale_a) * ld_scale(scale_b));
    if ((int)blockIdx.x >= main_blocks) {  // uniform per block
        partial = vec_partial;
        out = vec_out;
        pcol = 1; cols = 1; transpose = 0; ld_out = 1;
        mul = 1.0f / ld_scale(scale_a);
    }
    const int e = ((int)blockIdx.x >= main_blocks ? (int)blockIdx.x - main_blocks : (int)blockIdx.x) * 32 + threadIdx.x;
    const int total = rows * cols;
    float acc = 0.f;
    int r = 0, c = 0;
    if (e < total) {
        r = e / cols;
        c = e - r * cols;
        const float* p = partial + (size_t)r * pcol + c;
        const size_t stride = (size_t)prow * pcol;
        float a0 = 0.f, a1 = 0.f;
        int s = threadIdx.y;
        for (; s + 8 < S; s += 16) {
            a0 += p[(size_t)s * stride];
            a1 += p[(size_t)(s + 8) * stride];
        }
        if (s < S) a0 += p[(size_t)s * stride];
        acc = a0 + a1;
    }
    red[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && e < total) {
        float t = red[0][threadIdx.x];
#pragma unroll
        for (int y = 1; y < 8; ++y) t += red[y][threadIdx.x];
        t *= mul;
        if (transpose)
            out[(size_t)c * ld_out + r] = t;
        else
            out[(size_t)r * ld_out + c] = t;
    }
}

// Same reduction, four consecutive columns per thread (128-bit loads of the partial tiles): out[r][c..c+3] = mul * sum_s partial[s][r][c..c+3]
// for the non-transposed case with cols % 4 == 0 -- the weight-gradient tiles [256 x 256] x 74 splits of every update go through here.
// blockDim = (32, 8): 128 consecutive output elements per block, the S partials strided over threadIdx.y in the SAME fixed order as
// reduce_partials_kernel (bit-identical results).  Blocks beyond the matrix reduce the fused column-sum partials (scalar path).
__global__ void __launch_bounds__(256) reduce_partials_vec4_kernel(const float* __restrict__ partial, int S, int prow, int pcol, int rows, int cols,
                                                                   float* __restrict__ out, int ld_out, int main_blocks,
                                                                   const float* __restrict__ vec_partial, float* __restrict__ vec_out,
                                                                   const float* __restrict__ scale_a, const float* __restrict__ scale_b) {
    pdl_enter();
    __shared__ float4 red[8][33];
    if ((int)blockIdx.x >= main_blocks) {  // column-sum tail: one element per thread, as the scalar kernel
        const float mul = 1.0f / ld_scale(scale_a);
        const int e = ((int)blockIdx.x - main_blocks) * 32 + threadIdx.x;
        float acc = 0.f;
        if (e < rows) {
            const float* p = vec_partial + e;
            float a0 = 0.f, a1 = 0.f;
            int s = threadIdx.y;
            for (; s + 8 < S; s += 16) {
                a0 += p[(size_t)s * prow];
                a1 += p[(size_t)(s + 8) * prow];
            }
            if (s < S) a0 += p[(size_t)s * prow];
            acc = a0 + a1;
        }
        red[threadIdx.y][threadIdx.x].x = acc;
        __syncthreads();
        if (threadIdx.y == 0 && e < rows) {
            float t = red[0][threadIdx.x].x;
#pragma unroll
            for (int y = 1; y < 8; ++y) t += red[y][threadIdx.x].x;
            vec_out[e] = t * mul;
        }
        return;
    }
    const float mul = 1.0f / (ld_scale(scale_a) * ld_scale(scale_b));
    const int e4 = ((int)blockIdx.x * 32 + threadIdx.x) * 4;  // first of this thread's four output elements (row-major over rows x cols)
    const int total = rows * cols;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int r = 0, c = 0;
    if (e4 < total) {
        r = e4 / cols;
        c = e4 - r * cols;
        const float* p = partial + (size_t)r * pcol + c;
        const size_t stride = (size_t)prow * pcol;
        // this thread's partials (s = y, y + 8, ...; at most kRedMax of them) are loaded first -- independent 128-bit loads in flight
        // together -- and then added in the same alternating a0 / a1 order as the scalar kernel (bit-identical sums)
        constexpr int kRedMax = 12;
        float4 a0 = acc, a1 = acc;
        if (S <= 8 * kRedMax) {
            float4 v[kRedMax];
#pragma unroll
            for (int k = 0; k < kRedMax; ++k) {
                const int sk = threadIdx.y + 8 * k;
                v[k] = sk < S ? __ldcg(reinterpret_cast<const float4*>(p + (size_t)sk * stride)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int k = 0; k < kRedMax; ++k) {
                if ((int)threadIdx.y + 8 * k < S) {
                    if (k & 1) { a1.x += v[k].x; a1.y += v[k].y; a1.z += v[k].z; a1.w += v[k].w; }
                    else       { a0.x += v[k].x; a0.y += v[k].y; a0.z += v[k].z; a0.w += v[k].w; }
                }
            }
        } else {
            int s = threadIdx.y;
            for (; s + 8 < S; s += 16) {
                const float4 u = *reinterpret_cast<const float4*>(p + (size_t)s * stride);
                const float4 v = *reinterpret_cast<const float4*>(p + (size_t)(s + 8) * stride);
                a0.x += u.x; a0.y += u.y; a0.z += u.z; a0.w += u.w;
                a1.x += v.x; a1.y += v.y; a1.z += v.z; a1.w += v.w;
            }
            if (s < S) {
                const float4 u = *reinterpret_cast<const float4*>(p + (size_t)s * stride);
                a0.x += u.x; a0.y += u.y; a0.z += u.z; a0.w += u.w;
            }
        }
        acc = make_float4(a0.x + a1.x, a0.y + a1.y, a0.z + a1.z, a0.w + a1.w);
    }
    red[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && e4 < total) {
        float4 t = red[0][threadIdx.x];
#pragma unroll
        for (int y = 1; y < 8; ++y) {
            const float4 q = red[y][threadIdx.x];
            t.x += q.x; t.y += q.y; t.z += q.z; t.w += q.w;
        }
        *reinterpret_cast<float4*>(out + (size_t)r * ld_out + c) = make_float4(t.x * mul, t.y * mul, t.z * mul, t.w * mul);
    }
}

// column sums of a plane tensor: part[chunk][n] = sum over the chunk's rows and the P planes of G[p][m][n] (still scaled).
// blockDim = (32, 8): a thread owns 8 consecutive columns (one 16-byte load per plane per row) and every 8th row.
template <int FMT>
__global__ void __launch_bounds__(256) colsum_planes_kernel(const uint16_t* __restrict__ planes, long long plane_stride, int M, int ld, int N,
                                                            int rows_per_chunk, float* __restrict__ part) {
    using F = PlaneFmt<FMT>;
    __shared__ float red[8][32][9];
    const int n0 = (blockIdx.y * 32 + threadIdx.x) * 8;
    const int m0 = blockIdx.x * rows_per_chunk, m1 = min(M, m0 + rows_per_chunk);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (n0 < ld) {
        for (int m = m0 + threadIdx.y; m < m1; m += 8) {
            const size_t o = (size_t)m * ld + n0;
#pragma unroll
            for (int p = 0; p < F::P; ++p) F::add8(acc, __ldg(reinterpret_cast<const uint4*>(planes + p * plane_stride + o)));
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x][j] = acc[j];
    __syncthreads();
    if (threadIdx.y == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float t = 0.f;
#pragma unroll
            for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x][j];
            if (n0 + j < N) part[(size_t)blockIdx.x * N + n0 + j] = t;
        }
    }
}

// dU[b][h] = (1/scale) sum_j sum_p G[p][b*W + j][h]   (one block per b; blockDim = (32, 8), 8 columns per thread, j strided over y)
template <int FMT>
__global__ void __launch_bounds__(256) pairs_rowblock_sum_kernel(const uint16_t* __restrict__ planes, long long plane_stride, int W, int H,
                                                                 float* __restrict__ dU, const float* __restrict__ scale) {
    using F = PlaneFmt<FMT>;
    __shared__ float red[8][32][9];
    const int b = blockIdx.x;
    const int h0 = (blockIdx.y * 32 + threadIdx.x) * 8;
    const float inv = 1.0f / ld_scale(scale);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (h0 < H) {
        for (int j = threadIdx.y; j < W; j += 8) {
            const size_t o = ((size_t)b * W + j) * H + h0;
#pragma unroll
            for (int p = 0; p < F::P; ++p) F::add8(acc, __ldg(reinterpret_cast<const uint4*>(planes + p * plane_stride + o)));
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x][j] = acc[j];
    __syncthreads();
    if (threadIdx.y == 0 && h0 < H) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float t = 0.f;
#pragma unroll
            for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x][j];
            dU[(size_t)b * H + h0 + j] = t * inv;
        }
    }
}

// dU and the per-chunk partials of dV in ONE pass over the planes of dL/dh1 (|W| <= 64): block = (chunk of <= kPgrMaxB transitions, 256
// columns), thread (x, y) owns 8 columns and the weights j = y, y + 8, ...; the 8 y-partials of dU of every transition of the chunk are
// parked in shared memory and reduced after ONE barrier (same order as pairs_rowblock_sum_kernel), dV[j] accumulates over the
// transitions of the chunk in registers (its scale is removed by the final reduce_partials_kernel).
constexpr int kPgrMaxB = 8;
template <int FMT>
__global__ void __launch_bounds__(256, 2) pairs_grad_reduce_fused_kernel(const uint16_t* __restrict__ planes, long long plane_stride, int B, int W,
                                                                      int H, int b_per_chunk, float* __restrict__ dU, float* __restrict__ partV,
                                                                      const float* __restrict__ scale) {
    pdl_enter();
    using F = PlaneFmt<FMT>;
    extern __shared__ float red_dyn[];  // [kPgrMaxB][8][32][9]
    const int h0 = (blockIdx.y * 32 + threadIdx.x) * 8;
    const int b0 = blockIdx.x * b_per_chunk, b1 = min(B, b0 + b_per_chunk);
    const float inv = 1.0f / ld_scale(scale);
    float accV[8][8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int c = 0; c < 8; ++c) accV[k][c] = 0.f;
    for (int b = b0; b < b1; ++b) {
        float accU[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) accU[c] = 0.f;
        // four weight rows (x P planes) are loaded before any of them is used: with one row at a time the kernel had 32 bytes in flight per
        // thread and ran at a third of the HBM bandwidth (latency bound); predicated loads, no branches, same summation order
#pragma unroll
        for (int kk = 0; kk < 8; kk += 4) {
            uint4 ld[4][F::P];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int j = threadIdx.y + 8 * (kk + q);
                const bool ok = h0 < H && j < W;
                const size_t o = ok ? ((size_t)b * W + j) * H + h0 : 0;
#pragma unroll
                for (int p = 0; p < F::P; ++p)
                    ld[q][p] = ok ? __ldg(reinterpret_cast<const uint4*>(planes + p * plane_stride + o)) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float v[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) v[c] = 0.f;
#pragma unroll
                for (int p = 0; p < F::P; ++p) F::add8(v, ld[q][p]);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    accU[c] += v[c];
                    accV[kk + q][c] += v[c];
                }
            }
        }
        float* r = red_dyn + (((size_t)(b - b0) * 8 + threadIdx.y) * 32 + threadIdx.x) * 9;
#pragma unroll
        for (int c = 0; c < 8; ++c) r[c] = accU[c];
    }
    __syncthreads();
    if (h0 < H) {
        for (int bl = threadIdx.y; bl < b1 - b0; bl += 8) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float t = 0.f;
#pragma unroll
                for (int y = 0; y < 8; ++y) t += red_dyn[(((size_t)bl * 8 + y) * 32 + threadIdx.x) * 9 + c];
                dU[(size_t)(b0 + bl) * H + h0 + c] = t * inv;
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int j = threadIdx.y + 8 * k;
            if (j < W) {
                float* dst = partV + ((size_t)blockIdx.x * W + j) * H + h0;
                *reinterpret_cast<float4*>(dst) = make_float4(accV[k][0], accV[k][1], accV[k][2], accV[k][3]);
                *reinterpret_cast<float4*>(dst + 4) = make_float4(accV[k][4], accV[k][5], accV[k][6], accV[k][7]);
            }
        }
    }
}

// ---- power-of-two scale of a tensor from its largest magnitude ----------------------------------------------------------------
// scale = 2^(target_exp - e) with amax < 2^e, so that  2^(target_exp-1) <= scale * amax < 2^target_exp  (1 if the tensor is all zero).
__device__ __forceinline__ float scale_from_amax(float amax, int target_exp) {
    if (!(amax > 0.f) || !isfinite(amax)) return 1.0f;
    int e;
    (void)frexpf(amax, &e);
    int k = target_exp - e;
    k = k < -60 ? -60 : (k > 60 ? 60 : k);
    return ldexpf(1.0f, k);
}

// ws[0] = running max (bit pattern of a non-negative float), ws[1] = arrival counter; both zero on entry and zero again on exit
__global__ void __launch_bounds__(256) amax_scale_kernel(const float* __restrict__ src, long long n, int target_exp, float* __restrict__ scale_out,
                                                         unsigned int* __restrict__ ws) {
    pdl_enter();
    __shared__ float red[8];
    float m = 0.f;
    const long long n4 = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) ? (n >> 2) : 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    for (long long i = 4 * n4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(__ldg(src + i)));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        atomicMax(&ws[0], __float_as_uint(m));  // non-negative floats order like their bit patterns; max is order independent
        __threadfence();
        if (atomicAdd(&ws[1], 1u) == gridDim.x - 1) {
            __threadfence();
            const float amax = __uint_as_float(atomicExch(&ws[0], 0u));
            *scale_out = scale_from_amax(amax, target_exp);
            ws[1] = 0u;
        }
    }
}

// ---- fp32 -> planes (operands produced outside the GEMM epilogue: network inputs, weights, gradients) ---------------------------
template <int FMT>
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ src, int rows, int cols, int ld_src, int transpose,
                                                           uint16_t* __restrict__ dst, int rows_pad, int ldp, long long plane_stride,
                                                           const float* __restrict__ scale) {
    using F = PlaneFmt<FMT>;
    // dst[p][r][c] for r < rows_pad, c < ldp; source element (r, c) = transpose ? src[c * ld_src + r] : src[r * ld_src + c]
    const long long total = (long long)rows_pad * ldp;
    const float s = ld_scale(scale);
    float amax = 0.f;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(e / ldp), c = (int)(e - (long long)r * ldp);
        float x = 0.f;
        if (r < rows && c < cols) x = (transpose ? src[(size_t)c * ld_src + r] : src[(size_t)r * ld_src + c]) * s;
        uint16_t h[F::P];
        F::split1(x, h, amax);
#pragma unroll
        for (int p = 0; p < F::P; ++p) dst[p * plane_stride + e] = h[p];
    }
    if (FMT == MORL_FMT_F16X2) note_overflow(amax);
}

// non-transposed, ldp % 8 == 0: one thread converts 8 consecutive columns (two 128-bit loads when the source row allows it) and writes one
// 128-bit store per plane -- the gradient seed dL/dQ [65,536 x 24] of every step goes through here
template <int FMT>
__global__ void __launch_bounds__(256) split_planes_vec8_kernel(const float* __restrict__ src, int rows, int cols, int ld_src,
                                                                uint16_t* __restrict__ dst, int rows_pad, int ldp, long long plane_stride,
                                                                const float* __restrict__ scale) {
    pdl_enter();
    using F = PlaneFmt<FMT>;
    const int cpr = ldp >> 3;  // 8-column chunks per row
    const long long total = (long long)rows_pad * cpr;
    const bool vec_ok = (ld_src & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
    const float s = ld_scale(scale);
    float amax = 0.f;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(t / cpr), c0 = (int)(t - (long long)r * cpr) << 3;
        float x[8];
        if (r < rows && c0 + 8 <= cols && vec_ok) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ld_src + c0));
            const float4 b = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ld_src + c0 + 4));
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = (r < rows && c0 + k < cols) ? __ldg(src + (size_t)r * ld_src + c0 + k) : 0.f;
        }
        uint32_t pw[F::P][4];
#pragma unroll
        for (int k = 0; k < 8; k += 2) {
            uint32_t w[F::P];
            F::split2(x[k] * s, x[k + 1] * s, w, amax);
#pragma unroll
            for (int p = 0; p < F::P; ++p) pw[p][k >> 1] = w[p];
        }
        const size_t e = (size_t)r * ldp + c0;
#pragma unroll
        for (int p = 0; p < F::P; ++p) *reinterpret_cast<uint4*>(dst + p * plane_stride + e) = make_uint4(pw[p][0], pw[p][1], pw[p][2], pw[p][3]);
    }
    if (FMT == MORL_FMT_F16X2) note_overflow(amax);
}

// several small matrices (the weight matrices of a network, plain and transposed) in ONE launch: blockIdx.y selects the job.  Jobs with
// auto_scale != 0 derive their power-of-two scale from the largest |element| of their matrix in a one-block-per-job pre-pass
// (split_amax_multi_kernel, launched right before by the same entry point), which publishes it in *scale.
struct SplitJobs {
    MorlSplitJob job[MORL_SPLIT_MAX_JOBS];
};
__global__ void __launch_bounds__(1024) split_amax_multi_kernel(const __grid_constant__ SplitJobs jobs) {
    pdl_enter();
    __shared__ float red[32];
    const MorlSplitJob& j = jobs.job[blockIdx.x];
    if (!j.auto_scale || !j.scale) return;  // uniform per block
    const float* __restrict__ src = j.src;
    const int n_src = j.transpose ? j.cols : j.rows, k_src = j.transpose ? j.rows : j.cols;  // source matrix [n_src, k_src], row stride ld_src
    float m = 0.f;
    if (j.ld_src == k_src && (k_src & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15u) == 0) {  // dense: 128-bit loads
        const int n4 = (n_src * k_src) >> 2;
        for (int e = threadIdx.x; e < n4; e += blockDim.x) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(src) + e);
            m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
        }
    } else {
        for (int r = threadIdx.x / 32; r < n_src; r += blockDim.x / 32)
            for (int c = threadIdx.x & 31; c < k_src; c += 32) m = fmaxf(m, fabsf(__ldg(src + (size_t)r * j.ld_src + c)));
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = red[threadIdx.x];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
        if (threadIdx.x == 0) *j.scale = scale_from_amax(m, j.target_exp);
    }
}

template <int FMT>
__global__ void __launch_bounds__(256) split_planes_multi_kernel(const __grid_constant__ SplitJobs jobs) {
    pdl_enter();
    using F = PlaneFmt<FMT>;
    const MorlSplitJob& j = jobs.job[blockIdx.y];
    const float* __restrict__ src = j.src;
    uint16_t* __restrict__ dst = static_cast<uint16_t*>(j.dst_planes);
    const float s = j.scale ? *j.scale : 1.0f;  // (auto-scaled jobs: written by the pre-pass)
    const long long total = (long long)j.rows_pad * j.ldp;
    float amax = 0.f;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(e / j.ldp), c = (int)(e - (long long)r * j.ldp);
        float x = 0.f;
        if (r < j.rows && c < j.cols) x = (j.transpose ? src[(size_t)c * j.ld_src + r] : src[(size_t)r * j.ld_src + c]) * s;
        uint16_t h[F::P];
        F::split1(x, h, amax);
#pragma unroll
        for (int p = 0; p < F::P; ++p) dst[p * j.plane_stride + e] = h[p];
    }
    if (FMT == MORL_FMT_F16X2) note_overflow(amax);
}

// ---- separable first layer: h[b*W + j] = relu(u[b] + v[j]) straight into planes ------------------------------------------------
// PRODUCT: the product-conditioned first layer h[b*W + j] = u[b] * v[j] (one fp32 multiply, no activation: u and v are ReLU outputs)
template <int FMT, bool PRODUCT = false>
__global__ void __launch_bounds__(256) pairs_relu_split_kernel(const float* __restrict__ u, const float* __restrict__ v, int B, int W, int H,
                                                               uint16_t* __restrict__ dst, long long plane_stride, const float* __restrict__ scale,
                                                               uint32_t* __restrict__ bits_out) {
    pdl_enter();
    using F = PlaneFmt<FMT>;
    const int hv = H / 8;  // 8 columns per thread: two float4 loads per operand, one 16-byte store per plane
    const long long total = (long long)B * W * hv;
    const float s = ld_scale(scale);
    float amax = 0.f;
    const int lane = threadIdx.x & 31;
    // warp-uniform trip count (the bit words are assembled with shuffles): e0 = element of lane 0
    for (long long e0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x - lane); e0 < total; e0 += (long long)gridDim.x * blockDim.x) {
        const long long e = e0 + lane;
        const bool ok = e < total;
        const long long ee = ok ? e : 0;
        const int h8 = (int)(ee % hv);
        const long long row = ee / hv;
        const int b = (int)(row / W), j = (int)(row - (long long)b * W);
        const float4* up = reinterpret_cast<const float4*>(u + (size_t)b * H + 8 * h8);
        const float4* vp = reinterpret_cast<const float4*>(v + (size_t)j * H + 8 * h8);
        const float4 u0 = __ldg(up), u1 = __ldg(up + 1), v0 = __ldg(vp), v1 = __ldg(vp + 1);
        float x[8];
        if constexpr (PRODUCT) {
            x[0] = __fmul_rn(u0.x, v0.x); x[1] = __fmul_rn(u0.y, v0.y); x[2] = __fmul_rn(u0.z, v0.z); x[3] = __fmul_rn(u0.w, v0.w);
            x[4] = __fmul_rn(u1.x, v1.x); x[5] = __fmul_rn(u1.y, v1.y); x[6] = __fmul_rn(u1.z, v1.z); x[7] = __fmul_rn(u1.w, v1.w);
        } else {
            x[0] = u0.x + v0.x; x[1] = u0.y + v0.y; x[2] = u0.z + v0.z; x[3] = u0.w + v0.w;
            x[4] = u1.x + v1.x; x[5] = u1.y + v1.y; x[6] = u1.z + v1.z; x[7] = u1.w + v1.w;
        }
        uint32_t o[F::P][4];
        const uint32_t pos = pair_split8<FMT>(x, !PRODUCT, s, o, amax);  // bit t = (column 8 h8 + t is positive)
        if (ok) {
            const long long off = row * H + 8 * h8;
#pragma unroll
            for (int p = 0; p < F::P; ++p) *reinterpret_cast<uint4*>(dst + p * plane_stride + off) = make_uint4(o[p][0], o[p][1], o[p][2], o[p][3]);
        }
        if (bits_out) {
            // four consecutive threads (h8 = 4c .. 4c + 3; H % 32 == 0 keeps them in one aligned lane group) hold one 32-column word
            uint32_t wbits = pos << (8 * (lane & 3));
            wbits |= __shfl_xor_sync(0xffffffffu, wbits, 1);
            wbits |= __shfl_xor_sync(0xffffffffu, wbits, 2);
            if (ok && (lane & 3) == 0) {
                bits_out[(size_t)row * relu_bits_words(H) + relu_bits_word(32 * (h8 >> 2))] = wbits;
            }
        }
    }
    if (FMT == MORL_FMT_F16X2) note_overflow(amax);
}

// H = 256 form (the shape of the update): one warp per (transition b, quarter of the weight set), lane = 8 columns.  u[b] stays in
// registers for the warp's rows, v[j] comes from L1 / L2 (64 KB in total), four rows are in flight per iteration: half the load traffic of
// the element-indexed kernel above and no index arithmetic per element -- the kernel is a 67 MB write stream and nothing else.
template <int FMT>
__global__ void __launch_bounds__(256) pairs_relu_split_h256_kernel(const float* __restrict__ u, const float* __restrict__ v, int B, int W,
                                                                    uint16_t* __restrict__ dst, long long plane_stride,
                                                                    const float* __restrict__ scale, uint32_t* __restrict__ bits_out, int jsplit) {
    pdl_enter();
    using F = PlaneFmt<FMT>;
    constexpr int H = 256;
    const int lane = threadIdx.x & 31;
    const long long task = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (task >= (long long)B * jsplit) return;
    const int b = (int)(task / jsplit), js = (int)(task - (long long)b * jsplit);
    const int j0 = (int)((long long)W * js / jsplit), j1 = (int)((long long)W * (js + 1) / jsplit);
    const float s = ld_scale(scale);
    float amax = 0.f;
    const float4 u0 = __ldg(reinterpret_cast<const float4*>(u + (size_t)b * H + 8 * lane)),
                 u1 = __ldg(reinterpret_cast<const float4*>(u + (size_t)b * H + 8 * lane) + 1);
    const float uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
    for (int jb = j0; jb < j1; jb += 4) {
        float4 va[4], vb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int j = min(jb + q, j1 - 1);
            va[q] = __ldg(reinterpret_cast<const float4*>(v + (size_t)j * H + 8 * lane));
            vb[q] = __ldg(reinterpret_cast<const float4*>(v + (size_t)j * H + 8 * lane) + 1);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (jb + q >= j1) break;  // (warp-uniform)
            const float x[8] = {uu[0] + va[q].x, uu[1] + va[q].y, uu[2] + va[q].z, uu[3] + va[q].w,
                                uu[4] + vb[q].x, uu[5] + vb[q].y, uu[6] + vb[q].z, uu[7] + vb[q].w};
            uint32_t o[F::P][4];
            const uint32_t pos = pair_split8<FMT>(x, true, s, o, amax);
            const long long row = (long long)b * W + jb + q;
            const long long off = row * H + 8 * lane;
#pragma unroll
            for (int p = 0; p < F::P; ++p) *reinterpret_cast<uint4*>(dst + p * plane_stride + off) = make_uint4(o[p][0], o[p][1], o[p][2], o[p][3]);
            if (bits_out) {
                uint32_t wbits = pos << (8 * (lane & 3));
                wbits |= __shfl_xor_sync(0xffffffffu, wbits, 1);
                wbits |= __shfl_xor_sync(0xffffffffu, wbits, 2);
                if ((lane & 3) == 0) bits_out[(size_t)row * relu_bits_words(H) + relu_bits_word(8 * lane)] = wbits;
            }
        }
    }
    if (FMT == MORL_FMT_F16X2) note_overflow(amax);
}



static int make_plane_map_mn(CUtensorMap* map, int fmt, const void* base, int rows, int ld, long long plane_stride_elems) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return -1;
    const cuuint32_t P = (cuuint32_t)fmt_planes(fmt);
    const cuuint64_t dims[3] = {(cuuint64_t)ld, (cuuint64_t)rows, P};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)plane_stride_elems * 2};
    const cuuint32_t box[3] = {64, (cuuint32_t)kMnKT, P};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(map, fmt_tm_type(fmt), 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

// CTAs of a split-K weight-gradient launch (one per SM); morl_gemm_mn_workspace_bytes and the launcher must agree on it
static inline int mn_sm_count() {
    const int n = sm_count();
    return n <= 256 ? n : 132;  // (the column-sum tail of the workspace holds 256 splits)
}

static inline bool fmt_ok(int fmt) { return fmt == MORL_FMT_BF16X3 || fmt == MORL_FMT_F16X2; }

}  // namespace morl

extern "C" int morl_plane_overflow_count(int reset) {
    using namespace morl;
    unsigned int v = 0;
    cudaDeviceSynchronize();
    if (cudaMemcpyFromSymbol(&v, g_plane_overflow, sizeof(v)) != cudaSuccess) {
        (void)cudaGetLastError();
        set_error("morl_plane_overflow_count: no CUDA device");
        return MORL_ERR_NO_DEVICE;
    }
    if (reset) {
        const unsigned int z = 0;
        cudaMemcpyToSymbol(g_plane_overflow, &z, sizeof(z));
    }
    return (int)(v > 0x7fffffffu ? 0x7fffffffu : v);
}

extern "C" int morl_amax_scale_f32(const float* src, long long n, int target_exp, float* scale_out, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(src && scale_out && workspace, MORL_ERR_NULL, "morl_amax_scale_f32: NULL pointer argument");
    MORL_REQUIRE(n > 0 && target_exp >= -14 && target_exp <= 15, MORL_ERR_SHAPE, "morl_amax_scale_f32: bad n=%lld / target_exp=%d", n, target_exp);
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 132) blocks = 132;
    if (blocks < 1) blocks = 1;
    launch_k(amax_scale_kernel, dim3((int)blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), src, n, target_exp, scale_out, static_cast<unsigned int*>(workspace));
    return check_launch("morl_amax_scale_f32");
}

extern "C" size_t morl_gemm_mn_workspace_bytes(int M, int a_cols, int b_cols) {
    if (M <= 0 || a_cols <= 0 || b_cols <= 0) return 0;
    const int n_tiles = (a_cols + 127) / 128;
    const int NB = (b_cols + 63) / 64 * 64;
    int S = morl::mn_sm_count() / (n_tiles * (NB > 256 ? 2 : 1));
    if (S < 1) S = 1;
    int rps = ((M + S - 1) / S + 31) / 32 * 32;
    S = (M + rps - 1) / rps;
    return (size_t)S * n_tiles * 128 * NB * sizeof(float) + (size_t)256 * 256 * sizeof(float);  // tail: [S][n_tiles*128] column-sum partials
}

extern "C" int morl_gemm_planes_mn_f32(int fmt, const void* g_planes, long long g_plane_stride, int ldg, int g_cols, const float* g_scale,
                                       const void* h_planes, long long h_plane_stride, int ldh, int h_cols, const float* h_scale, int M,
                                       int transpose_out, float* out, int ld_out, float* colsum_out, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_gemm_planes_mn_f32: unknown plane format %d", fmt);
    MORL_REQUIRE(g_planes && h_planes && out && workspace, MORL_ERR_NULL, "morl_gemm_planes_mn_f32: NULL pointer argument");
    MORL_REQUIRE(M > 0 && g_cols > 0 && h_cols > 0, MORL_ERR_SHAPE, "morl_gemm_planes_mn_f32: bad shape M=%d g_cols=%d h_cols=%d", M, g_cols, h_cols);
    MORL_REQUIRE(ldg % 64 == 0 && ldh % 64 == 0 && ldh <= 512 && g_cols <= ldg && h_cols <= ldh, MORL_ERR_UNSUPPORTED,
                 "morl_gemm_planes_mn_f32: plane row lengths must be multiples of 64 (ldg=%d ldh=%d), ldh <= 512", ldg, ldh);
    const int n_tiles = (g_cols + 127) / 128;
    const int NB = (h_cols + 63) / 64 * 64;
    const int k_units = NB > 256 ? 2 : 1;  // (morl_gemm_mn_workspace_bytes derives the same S)
    MORL_REQUIRE(n_tiles * 128 <= ldg || ldg % 128 == 0 || n_tiles * 128 - ldg <= 64, MORL_ERR_UNSUPPORTED, "morl_gemm_planes_mn_f32: ldg=%d", ldg);
    int S = morl::mn_sm_count() / (n_tiles * k_units);
    if (S < 1) S = 1;
    const int rps = ((M + S - 1) / S + 31) / 32 * 32;
    S = (M + rps - 1) / rps;
    CUtensorMap tmA, tmB;
    int rc = make_plane_map_mn(&tmA, fmt, g_planes, M, ldg, g_plane_stride);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_planes_mn_f32: cuTensorMapEncodeTiled(G) failed (%d)", rc);
    rc = make_plane_map_mn(&tmB, fmt, h_planes, M, ldh, h_plane_stride);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_planes_mn_f32: cuTensorMapEncodeTiled(H) failed (%d)", rc);
    GemmMnArgs g;
    g.M = M; g.n_tiles = n_tiles; g.NB = NB; g.rows_per_split = rps; g.partial = static_cast<float*>(workspace);
    g.colsum_partial = colsum_out ? g.partial + (size_t)S * n_tiles * 128 * NB : nullptr;  // S * n_tiles * 128 <= 256 * 128 floats: the 256 KB tail
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    MORL_DISPATCH_FMT(fmt, {
        using F = PlaneFmt<kFmt>;
        const size_t smem = (size_t)F::kStagesMn * (6u * F::P * kMnKT * 128u) + 256 + 1024 + 64 + 1024 + 4096;
        set_smem_limit_once<gemm_planes_mn_kernel<kFmt>>(smem);
        launch_k(gemm_planes_mn_kernel<kFmt>, dim3(n_tiles * k_units * S), dim3(kGemmThreads), smem, st, tmA, tmB, g);
    });
    rc = check_launch("morl_gemm_planes_mn_f32");
    if (rc) return rc;
    const int total = g_cols * h_cols;
    const int main_blocks = (total + 31) / 32, vec_blocks = colsum_out ? (g_cols + 31) / 32 : 0;
    if (!transpose_out && h_cols % 4 == 0 && ld_out % 4 == 0 && aligned16(out)) {
        const int mb4 = (total / 4 + 31) / 32;
        launch_k(reduce_partials_vec4_kernel, dim3(mb4 + vec_blocks), dim3(dim3(32, 8)), 0, st, g.partial, S, n_tiles * 128, NB, g_cols, h_cols, out, ld_out, mb4,
                                                                              g.colsum_partial, colsum_out, g_scale, h_scale);
        return check_launch("morl_gemm_planes_mn_f32(reduce)");
    }
    launch_k(reduce_partials_kernel, dim3(main_blocks + vec_blocks), dim3(dim3(32, 8)), 0, st, g.partial, S, n_tiles * 128, NB, g_cols, h_cols, transpose_out, out, ld_out,
                                                                             main_blocks, g.colsum_partial, colsum_out, g_scale, h_scale);
    return check_launch("morl_gemm_planes_mn_f32(reduce)");
}

// Row chunks of the split column sums: each chunk writes one row of partials to the workspace, reduced in a fixed order afterwards.
constexpr int kPgrFusedChunks = 296;   // morl_pairs_grad_reduce_planes, one-pass form
constexpr int kPgrTwoPassChunks = 74;  // morl_pairs_grad_reduce_planes, two-pass form

// Transitions per chunk of the one-pass pairs_grad_reduce (at most kPgrMaxB, at most kPgrFusedChunks chunks), or 0 when the two-pass
// form runs instead.
static int pgr_fused_rows_per_chunk(int B, int W) {
    if (W > 64) return 0;
    int bpc = (B + kPgrFusedChunks - 1) / kPgrFusedChunks;
    if (bpc > morl::kPgrMaxB) bpc = morl::kPgrMaxB;
    return (B + bpc - 1) / bpc <= kPgrFusedChunks ? bpc : 0;
}

extern "C" size_t morl_pairs_grad_reduce_workspace_bytes(int B, int W, int H) {
    if (B <= 0 || W <= 0 || H <= 0) return 0;
    return (size_t)(pgr_fused_rows_per_chunk(B, W) ? kPgrFusedChunks : kPgrTwoPassChunks) * W * H * sizeof(float);
}

extern "C" int morl_pairs_grad_reduce_planes(int fmt, const void* planes, long long plane_stride, const float* scale, int B, int W, int H, float* dU,
                                             float* dV, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_pairs_grad_reduce_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(planes && dU && dV && workspace, MORL_ERR_NULL, "morl_pairs_grad_reduce_planes: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && H > 0 && H % 8 == 0 && plane_stride % 8 == 0, MORL_ERR_SHAPE, "morl_pairs_grad_reduce_planes: bad shape B=%d W=%d H=%d", B, W, H);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint16_t* pl = static_cast<const uint16_t*>(planes);
    if (const int bpc = pgr_fused_rows_per_chunk(B, W)) {
        // one pass: dU directly, dV as per-chunk partials [chunks][W*H] reduced in a fixed order
        const int nchf = (B + bpc - 1) / bpc;
        const int Nf = W * H;
        float* partf = static_cast<float*>(workspace);
        const size_t smemf = (size_t)kPgrMaxB * 8 * 32 * 9 * sizeof(float);  // 73,728 B
        MORL_DISPATCH_FMT(fmt, {
            set_smem_limit_once<pairs_grad_reduce_fused_kernel<kFmt>>(smemf);
            launch_k(pairs_grad_reduce_fused_kernel<kFmt>, dim3(dim3((unsigned)nchf, (unsigned)((H + 255) / 256))), dim3(dim3(32, 8)), smemf, st, pl, plane_stride, B, W,
                                                                                                                                 H, bpc, dU, partf, scale);
        });
        int rcf = check_launch("morl_pairs_grad_reduce_planes(fused)");
        if (rcf) return rcf;
        launch_k(reduce_partials_kernel, dim3((Nf + 31) / 32), dim3(dim3(32, 8)), 0, st, partf, nchf, 1, Nf, 1, Nf, 0, dV, Nf, 1 << 30, nullptr, nullptr, scale, nullptr);
        return check_launch("morl_pairs_grad_reduce_planes(reduce)");
    }
    // dU[b] = sum over the W rows of transition b
    MORL_DISPATCH_FMT(fmt, (pairs_rowblock_sum_kernel<kFmt><<<dim3((unsigned)B, (unsigned)((H + 255) / 256)), dim3(32, 8), 0, st>>>(pl, plane_stride, W, H,
                                                                                                                                     dU, scale)));
    int rc = check_launch("morl_pairs_grad_reduce_planes(dU)");
    if (rc) return rc;
    // dV[j] = sum over b: column sums of the [B, W*H] view
    const int N = W * H;
    const int chunks = kPgrTwoPassChunks;
    const int rpc = (B + chunks - 1) / chunks;
    const int nch = (B + rpc - 1) / rpc;
    float* part = static_cast<float*>(workspace);
    MORL_DISPATCH_FMT(fmt, (colsum_planes_kernel<kFmt><<<dim3((unsigned)nch, (unsigned)((N + 255) / 256)), dim3(32, 8), 0, st>>>(pl, plane_stride, B, N, N,
                                                                                                                                  rpc, part)));
    rc = check_launch("morl_pairs_grad_reduce_planes(dV)");
    if (rc) return rc;
    launch_k(reduce_partials_kernel, dim3((N + 31) / 32), dim3(dim3(32, 8)), 0, st, part, nch, 1, N, 1, N, 0, dV, N, 1 << 30, nullptr, nullptr, scale, nullptr);
    return check_launch("morl_pairs_grad_reduce_planes(reduce)");
}

extern "C" int morl_split_planes(int fmt, const float* src, int rows, int cols, int ld_src, int transpose, void* dst_planes, int rows_pad, int ldp,
                                 long long plane_stride, const float* scale, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_split_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(src && dst_planes, MORL_ERR_NULL, "morl_split_planes: NULL pointer argument");
    MORL_REQUIRE(rows > 0 && cols > 0 && rows_pad >= rows && ldp >= cols && ld_src > 0, MORL_ERR_SHAPE,
                 "morl_split_planes: bad shape rows=%d cols=%d rows_pad=%d ldp=%d", rows, cols, rows_pad, ldp);
    MORL_REQUIRE(plane_stride >= (long long)rows_pad * ldp, MORL_ERR_SHAPE, "morl_split_planes: plane_stride too small");
    const long long total = (long long)rows_pad * ldp;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint16_t* dst = static_cast<uint16_t*>(dst_planes);
    if (!transpose && (ldp & 7) == 0 && (plane_stride & 7) == 0 && (reinterpret_cast<uintptr_t>(dst_planes) & 15u) == 0) {
        const long long chunks = total >> 3;
        long long vb = (chunks + 255) / 256;
        if (vb > 132 * 8) vb = 132 * 8;
        MORL_DISPATCH_FMT(fmt, (launch_k(split_planes_vec8_kernel<kFmt>, dim3((int)vb), dim3(256), 0, st, src, rows, cols, ld_src, dst, rows_pad, ldp, plane_stride, scale)));
        return check_launch("morl_split_planes(vec8)");
    }
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    MORL_DISPATCH_FMT(fmt, (split_planes_kernel<kFmt><<<(int)blocks, 256, 0, st>>>(src, rows, cols, ld_src, transpose, dst, rows_pad, ldp, plane_stride, scale)));
    return check_launch("morl_split_planes");
}

extern "C" int morl_split_planes_multi(int fmt, const MorlSplitJob* jobs, int n_jobs, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_split_planes_multi: unknown plane format %d", fmt);
    MORL_REQUIRE(jobs, MORL_ERR_NULL, "morl_split_planes_multi: NULL pointer argument");
    MORL_REQUIRE(n_jobs > 0 && n_jobs <= MORL_SPLIT_MAX_JOBS, MORL_ERR_SHAPE, "morl_split_planes_multi: n_jobs=%d out of range", n_jobs);
    SplitJobs sj;
    memset(&sj, 0, sizeof(sj));
    long long max_total = 0;
    for (int i = 0; i < n_jobs; ++i) {
        const MorlSplitJob& j = jobs[i];
        MORL_REQUIRE(j.src && j.dst_planes, MORL_ERR_NULL, "morl_split_planes_multi: job %d has a NULL pointer", i);
        MORL_REQUIRE(j.rows > 0 && j.cols > 0 && j.rows_pad >= j.rows && j.ldp >= j.cols && j.ld_src > 0 &&
                         j.plane_stride >= (long long)j.rows_pad * j.ldp,
                     MORL_ERR_SHAPE, "morl_split_planes_multi: job %d bad shape rows=%d cols=%d rows_pad=%d ldp=%d", i, j.rows, j.cols, j.rows_pad, j.ldp);
        MORL_REQUIRE(!j.auto_scale || (j.scale && j.target_exp >= -14 && j.target_exp <= 15), MORL_ERR_SHAPE,
                     "morl_split_planes_multi: job %d auto_scale needs a scale pointer and -14 <= target_exp <= 15 (got %d)", i, j.target_exp);
        sj.job[i] = j;
        const long long t = (long long)j.rows_pad * j.ldp;
        if (t > max_total) max_total = t;
    }
    long long bx = (max_total + 255) / 256;
    if (bx > 132) bx = 132;
    bool any_auto = false;
    for (int i = 0; i < n_jobs; ++i) any_auto = any_auto || (jobs[i].auto_scale && jobs[i].scale);
    if (any_auto) {
        launch_k(split_amax_multi_kernel, dim3(n_jobs), dim3(1024), 0, static_cast<cudaStream_t>(stream), sj);
        int rca = check_launch("morl_split_planes_multi(amax)");
        if (rca) return rca;
    }
    MORL_DISPATCH_FMT(fmt, (launch_k(split_planes_multi_kernel<kFmt>, dim3(dim3((unsigned)bx, (unsigned)n_jobs)), dim3(256), 0, static_cast<cudaStream_t>(stream), sj)));
    return check_launch("morl_split_planes_multi");
}

extern "C" int morl_pairs_relu_split_planes(int fmt, const float* u, const float* v, int B, int W, int H, void* dst_planes, long long plane_stride,
                                            const float* scale, void* relu_bits_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_pairs_relu_split_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(u && v && dst_planes, MORL_ERR_NULL, "morl_pairs_relu_split_planes: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && H > 0 && H % 8 == 0 && plane_stride % 8 == 0 && plane_stride >= (long long)B * W * H, MORL_ERR_SHAPE,
                 "morl_pairs_relu_split_planes: bad shape B=%d W=%d H=%d", B, W, H);
    const long long total = (long long)B * W * (H / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (relu_bits_out)
        MORL_REQUIRE(H % 32 == 0 && H <= 512 && aligned16(relu_bits_out), MORL_ERR_SHAPE,
                     "morl_pairs_relu_split_planes: ReLU bit masks need H %% 32 == 0, H <= 512 (H=%d)", H);
    if (H == 256) {
        const int jsplit = W >= 16 ? 4 : 1;
        const long long tasks = (long long)B * jsplit;
        MORL_DISPATCH_FMT(fmt, (launch_k(pairs_relu_split_h256_kernel<kFmt>, dim3((unsigned)((tasks + 7) / 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                                         u, v, B, W, static_cast<uint16_t*>(dst_planes), plane_stride, scale, static_cast<uint32_t*>(relu_bits_out), jsplit)));
        return check_launch("morl_pairs_relu_split_planes(h256)");
    }
    MORL_DISPATCH_FMT(fmt, (launch_k(pairs_relu_split_kernel<kFmt>, dim3((int)blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), 
                               u, v, B, W, H, static_cast<uint16_t*>(dst_planes), plane_stride, scale, static_cast<uint32_t*>(relu_bits_out))));
    return check_launch("morl_pairs_relu_split_planes");
}

extern "C" int morl_pairs_product_split_planes(int fmt, const float* u, const float* v, int B, int P, int H, void* dst_planes, long long plane_stride,
                                               const float* scale, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_pairs_product_split_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(u && v && dst_planes, MORL_ERR_NULL, "morl_pairs_product_split_planes: NULL pointer argument");
    MORL_REQUIRE(B > 0 && P > 0 && H > 0 && H % 8 == 0 && plane_stride % 8 == 0 && plane_stride >= (long long)B * P * H, MORL_ERR_SHAPE,
                 "morl_pairs_product_split_planes: bad shape B=%d P=%d H=%d", B, P, H);
    MORL_REQUIRE(aligned16(u) && aligned16(v) && aligned16(dst_planes), MORL_ERR_ALIGN, "morl_pairs_product_split_planes: operands must be 16-byte aligned");
    const long long total = (long long)B * P * (H / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    MORL_DISPATCH_FMT(fmt, (launch_k(pairs_relu_split_kernel<kFmt, true>, dim3((int)blocks), dim3(256), 0, static_cast<cudaStream_t>(stream),
                                     u, v, B, P, H, static_cast<uint16_t*>(dst_planes), plane_stride, scale, static_cast<uint32_t*>(nullptr))));
    return check_launch("morl_pairs_product_split_planes");
}

// Diagnostics: cycle counters of the K-major GEMM roles, accumulated over all CTAs and launches since the last reset
// (only when MORL_GEMM_STATS=1 was set before the first GEMM call).
extern "C" int morl_debug_gemm_stats(unsigned long long* out8, int reset) {
    using namespace morl;
    MORL_REQUIRE(out8, MORL_ERR_NULL, "morl_debug_gemm_stats: NULL pointer argument");
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out8, g_gemm_stats, 8 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        cudaMemcpyToSymbol(g_gemm_stats, z, sizeof(z));
    }
    return check_launch("morl_debug_gemm_stats");
}

namespace morl {
template <int FMT, int SPLIT, int EPI = kEpiPlain>
static int launch_gemm_planes(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmArgs& g, int sms, cudaStream_t st) {
    constexpr size_t smem = KPlan<FMT>::kBytes;
    set_smem_limit_once<gemm_planes_kernel<FMT, SPLIT, EPI>>(smem);
    constexpr int kUnitN = SPLIT ? 128 : 256;  // column units per tile: as gemm_planes_kernel
    const int n_work = (g.M + kGemmBM - 1) / kGemmBM * ((g.N_pad + kUnitN - 1) / kUnitN);
    launch_k_pdl(true, gemm_planes_kernel<FMT, SPLIT, EPI>, dim3(n_work < sms ? n_work : sms), dim3(kGemmThreads), smem, st, tmA, tmB, tmC, g);
    return check_launch(EPI == kEpiLn ? "morl_gemm_planes_ln_f32" : "morl_gemm_planes_f32");
}

// the LayerNorm / dropout part of a morl_gemm_planes_ln_f32 call (nullptr: morl_gemm_planes_f32)
struct LnDropArgs {
    int ln;
    float eps;
    const float *gamma, *beta;
    const unsigned long long* seed;
    const unsigned int* offset;
    unsigned int salt, thr;
    float scale;
    void* bits;
};

static int gemm_planes_impl(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                            long long b_plane_stride, const float* b_scale, int M, int N, int N_pad, int K, const float* bias, int relu,
                            float* c_f32, int ldc, void* c_planes, int ldp, long long c_plane_stride, const float* c_scale, int reverse_tiles,
                            int split_accumulators, const void* relu_bits_in, void* relu_bits_out, const LnDropArgs* lnd, const char* name, void* stream) {
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "%s: unknown plane format %d", name, fmt);
    MORL_REQUIRE(a_planes && b_planes && (c_f32 || c_planes), MORL_ERR_NULL, "%s: NULL pointer argument", name);
    MORL_REQUIRE(M > 0 && N > 0 && K > 0 && N_pad >= N, MORL_ERR_SHAPE, "%s: bad shape M=%d N=%d N_pad=%d K=%d", name, M, N, N_pad, K);
    const int BK = fmt_bk(fmt);
    MORL_REQUIRE(K % BK == 0 && N_pad % 32 == 0 && N_pad <= 512, MORL_ERR_UNSUPPORTED,
                 "%s: need K %% %d == 0, N_pad %% 32 == 0, N_pad <= 512 (K=%d N_pad=%d)", name, BK, K, N_pad);
    MORL_REQUIRE(aligned16(a_planes) && aligned16(b_planes), MORL_ERR_ALIGN, "%s: operand planes must be 16-byte aligned", name);
    MORL_REQUIRE(aligned16(relu_bits_in) && aligned16(relu_bits_out), MORL_ERR_ALIGN, "%s: ReLU bit masks must be 16-byte aligned", name);
    if (c_planes)
        MORL_REQUIRE(ldp % 32 == 0 && ldp >= N && ldp <= N_pad && aligned16(c_planes) && c_plane_stride % 8 == 0, MORL_ERR_SHAPE,
                     "%s: ldp=%d must be a multiple of 32 with N <= ldp <= N_pad", name, ldp);
    CUtensorMap tmA, tmB;
    int rc = make_plane_map(&tmA, fmt, a_planes, M, K, a_plane_stride, kGemmBM, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(A) failed (%d)", name, rc);
    rc = make_plane_map(&tmB, fmt, b_planes, N_pad, K, b_plane_stride, kGemmBoxN, BK, true);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(B) failed (%d)", name, rc);
    CUtensorMap tmC;
    memset(&tmC, 0, sizeof(tmC));
    if (c_planes) {  // store map of the re-split output: [P][M][ldp], box 32 cols x 16 rows x P planes (64-byte swizzle)
        rc = make_plane_map(&tmC, fmt, c_planes, M, ldp, c_plane_stride, 16, 32);
        MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(C) failed (%d)", name, rc);
    }
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = N; g.N_pad = N_pad; g.K = K;
    g.bias = bias; g.c_f32 = c_f32; g.ldc = ldc;
    g.c_planes = c_planes; g.ldp = ldp; g.plane_stride = c_plane_stride;
    g.relu = relu;
    g.bits_in = static_cast<const uint32_t*>(relu_bits_in); g.bits_out = static_cast<uint32_t*>(relu_bits_out);
    g.bits_ld = relu_bits_words(N_pad);  // every 32-column chunk below N_pad has its word, padding chunks included
    {
        // TMA ring: A box + B rows per stage; a narrow B (the output layer: N_pad = 32) leaves room for a deeper ring, which is what
        // keeps enough bytes in flight per SM when a tile is four A boxes and almost no tensor work
        const uint32_t rowb = (uint32_t)BK * 2u, P = (uint32_t)fmt_planes(fmt);
        const uint32_t a_box = P * (uint32_t)kGemmBM * rowb;
        const uint32_t n_unit = N_pad > 256 ? 256u : (uint32_t)N_pad;  // B rows of one column unit (outputs wider than 256: two units)
        const uint32_t b_box = (P * n_unit * rowb + 1023u) & ~1023u;
        const uint32_t room = fmt == MORL_FMT_F16X2 ? KPlan<MORL_FMT_F16X2>::kOffC : KPlan<MORL_FMT_BF16X3>::kOffC;
        int n_st = (int)(room / (a_box + b_box));
        if (n_st > 8) n_st = 8;
        g.n_stages = n_st;
        g.b_stage = b_box;
    }
    g.a_scale = a_scale; g.b_scale = b_scale; g.c_scale = c_scale;
    g.reverse = reverse_tiles ? 1 : 0;
    static const bool want_stats = [] { const char* e = getenv("MORL_GEMM_STATS"); return e && e[0] == '1'; }();
    g.stats = nullptr;
    if (want_stats) {
        void* sp = nullptr;
        cudaGetSymbolAddress(&sp, g_gemm_stats);
        g.stats = static_cast<unsigned long long*>(sp);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int sms = sm_count();
    if (lnd) {
        g.ln = lnd->ln; g.ln_eps = lnd->eps; g.ln_gamma = lnd->gamma; g.ln_beta = lnd->beta;
        g.drop_seed = lnd->seed; g.drop_offset = lnd->offset; g.drop_salt = lnd->salt; g.drop_thr = lnd->thr; g.drop_scale = lnd->scale;
        g.drop_bits = static_cast<uint32_t*>(lnd->bits);
        return fmt == MORL_FMT_F16X2 ? launch_gemm_planes<MORL_FMT_F16X2, 0, kEpiLn>(tmA, tmB, tmC, g, sms, st)
                                     : launch_gemm_planes<MORL_FMT_BF16X3, 0, kEpiLn>(tmA, tmB, tmC, g, sms, st);
    }
    // accumulator mode (see gemm_planes_kernel): per call
    if (fmt == MORL_FMT_F16X2)
        return split_accumulators ? launch_gemm_planes<MORL_FMT_F16X2, 1>(tmA, tmB, tmC, g, sms, st) : launch_gemm_planes<MORL_FMT_F16X2, 0>(tmA, tmB, tmC, g, sms, st);
    return split_accumulators ? launch_gemm_planes<MORL_FMT_BF16X3, 1>(tmA, tmB, tmC, g, sms, st) : launch_gemm_planes<MORL_FMT_BF16X3, 0>(tmA, tmB, tmC, g, sms, st);
}

__global__ void philox_advance_kernel(unsigned int* offset, unsigned int inc) {
    pdl_enter();
    *offset += inc;
}
}  // namespace morl

extern "C" int morl_gemm_planes_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                                    long long b_plane_stride, const float* b_scale, int M, int N, int N_pad, int K, const float* bias, int relu,
                                    float* c_f32, int ldc, void* c_planes, int ldp, long long c_plane_stride, const float* c_scale, int reverse_tiles,
                                    int split_accumulators, const void* relu_bits_in, void* relu_bits_out, void* stream) {
    return morl::gemm_planes_impl(fmt, a_planes, a_plane_stride, a_scale, b_planes, b_plane_stride, b_scale, M, N, N_pad, K, bias, relu, c_f32, ldc,
                                  c_planes, ldp, c_plane_stride, c_scale, reverse_tiles, split_accumulators, relu_bits_in, relu_bits_out, nullptr,
                                  "morl_gemm_planes_f32", stream);
}

extern "C" int morl_gemm_planes_ln_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                                       long long b_plane_stride, const float* b_scale, int M, int N, int K, const float* bias, int layer_norm,
                                       const float* ln_gamma, const float* ln_beta, float ln_eps, float drop_p, const unsigned long long* drop_seed,
                                       const unsigned int* drop_offset, unsigned int drop_salt, float* c_f32, int ldc, void* c_planes, int ldp,
                                       long long c_plane_stride, const float* c_scale, int reverse_tiles, void* drop_bits_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_gemm_planes_ln_f32: unknown plane format %d", fmt);
    MORL_REQUIRE(N > 0 && N <= 256 && N % 32 == 0, MORL_ERR_UNSUPPORTED, "morl_gemm_planes_ln_f32: need N %% 32 == 0 and N <= 256 (N=%d)", N);
    MORL_REQUIRE(!(drop_p < 0.f) && drop_p < 1.f, MORL_ERR_SHAPE, "morl_gemm_planes_ln_f32: dropout probability %g outside [0, 1)", (double)drop_p);
    MORL_REQUIRE(!layer_norm || ln_eps > 0.f, MORL_ERR_SHAPE, "morl_gemm_planes_ln_f32: LayerNorm eps must be positive (got %g)", (double)ln_eps);
    MORL_REQUIRE((drop_seed == nullptr) == (drop_offset == nullptr), MORL_ERR_NULL, "morl_gemm_planes_ln_f32: dropout needs both the seed and the offset");
    MORL_REQUIRE(drop_seed || !drop_bits_out, MORL_ERR_NULL, "morl_gemm_planes_ln_f32: a keep mask needs dropout (seed and offset)");
    MORL_REQUIRE(aligned16(drop_bits_out), MORL_ERR_ALIGN, "morl_gemm_planes_ln_f32: the keep mask must be 16-byte aligned");
    LnDropArgs a;
    a.ln = layer_norm ? 1 : 0; a.eps = ln_eps; a.gamma = ln_gamma; a.beta = ln_beta;
    a.seed = drop_seed; a.offset = drop_offset; a.salt = drop_salt;
    const double t = rint((double)drop_p * 4294967296.0);  // keep iff draw >= round(p 2^32); p < 1 keeps it below 2^32
    a.thr = t >= 4294967295.0 ? 4294967295u : (unsigned int)t;
    a.scale = (float)(1.0 / (1.0 - (double)drop_p));
    a.bits = drop_bits_out;
    return gemm_planes_impl(fmt, a_planes, a_plane_stride, a_scale, b_planes, b_plane_stride, b_scale, M, N, N, K, bias, 1, c_f32, ldc, c_planes, ldp,
                            c_plane_stride, c_scale, reverse_tiles, 0, nullptr, nullptr, &a, "morl_gemm_planes_ln_f32", stream);
}

extern "C" int morl_philox_advance(unsigned int* offset, unsigned int inc, void* stream) {
    using namespace morl;
    MORL_REQUIRE(offset, MORL_ERR_NULL, "morl_philox_advance: NULL pointer argument");
    launch_k(philox_advance_kernel, dim3(1), dim3(1), 0, static_cast<cudaStream_t>(stream), offset, inc);
    return check_launch("morl_philox_advance");
}


namespace morl {
// The ChainArgs of a chain launch, and the weight and output tensor maps of its jobs.  Job (c, l) = layer l of chain c reads the weight
// planes w_planes[job] ([P][256][K]; layer 0: [P][256][k_first]) and, when bit job of `store` is set, writes its output to
// acts[c (n_layers + 1) + l + 1] ([P][M][256]).  f16x2 runs on gemm_chain_resident_kernel (weight boxes of 256 rows, output boxes of one
// plane), bf16x3 on gemm_chain_kernel (weight boxes of 32 rows, output boxes of all planes).
static int set_chain_args(ChainArgs& g, CUtensorMap* B, CUtensorMap* C, int fmt, int n_chains, int n_layers, int M, int K, int k_first,
                          const void* const* acts, long long act_plane_stride, const float* act_scale, uint32_t store, const void* const* w_planes,
                          long long w_plane_stride, const float* const* w_scales, const float* const* biases, int relu,
                          const void* const* relu_bits_in, void* const* relu_bits_out, const char* name) {
    const bool resident = fmt == MORL_FMT_F16X2;
    const int BK = resident ? ResPlan::BK : fmt_bk(fmt);
    g.M = M; g.K = K; g.k_first = k_first; g.n_chains = n_chains; g.n_layers = n_layers; g.a_scale = act_scale; g.relu = relu ? 1 : 0;
    for (int c = 0; c < n_chains; ++c)
        for (int l = 0; l < n_layers; ++l) {
            const int job = c * n_layers + l;
            const int kj = l == 0 ? k_first : K;
            const long long w_stride = l == 0 ? (long long)256 * k_first : w_plane_stride;
            MORL_REQUIRE(w_planes[job] && aligned16(w_planes[job]), MORL_ERR_NULL, "%s: NULL or misaligned weight planes (chain %d, layer %d)", name, c, l);
            int rc = make_plane_map(&B[job], fmt, w_planes[job], 256, kj, w_stride, resident ? 256 : kGemmBoxN, BK, true);
            MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(B) failed (%d)", name, rc);
            if ((store >> job) & 1u) {
                const void* out = acts[c * (n_layers + 1) + l + 1];
                MORL_REQUIRE(out && aligned16(out), MORL_ERR_NULL, "%s: NULL or misaligned output planes (chain %d, layer %d)", name, c, l);
                rc = make_plane_map(&C[job], fmt, out, M, 256, act_plane_stride, 16, 32, resident);
                MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(C) failed (%d)", name, rc);
            }
            g.bias[job] = biases ? biases[job] : nullptr;
            g.b_scale[job] = w_scales ? w_scales[job] : nullptr;
            g.bits_out[job] = relu_bits_out ? static_cast<uint32_t*>(relu_bits_out[job]) : nullptr;
            g.bits_in[job] = relu_bits_in ? static_cast<const uint32_t*>(relu_bits_in[job]) : nullptr;
            MORL_REQUIRE(aligned16(g.bits_out[job]) && aligned16(g.bits_in[job]), MORL_ERR_ALIGN, "%s: ReLU bit masks must be 16-byte aligned", name);
        }
    return MORL_OK;
}

// Launch of gemm_chain_resident_kernel.  g: store and (pair mode) u / v / W set by the caller; in[c]: planes-mode input of chain c
// ([P][M][k_first], nullptr in pair mode); acts: as set_chain_args.
static int launch_chain_resident(ResChainArgs& g, int n_chains, int n_layers, int k_first, const void* const* in, const void* const* acts,
                                 long long act_plane_stride, const float* act_scale, const void* const* w_planes, long long w_plane_stride,
                                 const float* const* w_scales, const float* const* biases, int relu, const void* const* relu_bits_in,
                                 void* const* relu_bits_out, int M, int K, const char* name, void* stream) {
    constexpr int fmt = MORL_FMT_F16X2;
    ResChainMaps maps;
    memset(&maps, 0, sizeof(maps));
    const int rc = set_chain_args(g, maps.B, maps.C, fmt, n_chains, n_layers, M, K, k_first, acts, act_plane_stride, act_scale, g.store, w_planes,
                                  w_plane_stride, w_scales, biases, relu, relu_bits_in, relu_bits_out, name);
    if (rc) return rc;
    for (int c = 0; c < n_chains && !g.u[0]; ++c) {
        MORL_REQUIRE(in[c] && aligned16(in[c]), MORL_ERR_NULL, "%s: NULL or misaligned input planes (chain %d)", name, c);
        // [P][M][k_first] (plane stride M * k_first), box P x 128 rows x 32
        const int rca = make_plane_map(&maps.A[c], fmt, in[c], M, k_first, (long long)M * k_first, kGemmBM, ResPlan::BK);
        MORL_REQUIRE(rca == 0, MORL_ERR_NO_DEVICE, "%s: cuTensorMapEncodeTiled(A) failed (%d)", name, rca);
    }
    static const bool want_stats = [] { const char* e = getenv("MORL_GEMM_STATS"); return e && e[0] == '1'; }();
    if (want_stats) {
        void* sp = nullptr;
        cudaGetSymbolAddress(&sp, g_gemm_stats);
        g.stats = static_cast<unsigned long long*>(sp);
    }
    const int sms = sm_count();
    const int n_tiles = (M + kGemmBM - 1) / kGemmBM;
    constexpr size_t smem = ResPlan::kBytes;
    set_smem_limit_once<gemm_chain_resident_kernel>(smem);
    launch_k_pdl(true, gemm_chain_resident_kernel, dim3(n_tiles < sms ? n_tiles : sms), dim3(kGemmThreads), smem,
                 static_cast<cudaStream_t>(stream), maps, g);
    return check_launch(name);
}
}  // namespace morl

extern "C" int morl_gemm_chain_supported(int fmt, int M, int K) {
    using namespace morl;
    return fmt_ok(fmt) && M >= 2 * kGemmBM && K == 256;
}

// Several 256-wide hidden layers (Linear + ReLU, planes in / planes out) of one or two networks in ONE persistent launch: job (c, l) computes
// act[c][l+1] = relu(act[c][l] . W[c][l]^T + bias[c][l]) exactly as morl_gemm_planes_f32 does (bit-identical), but a CTA takes its row tiles
// through all layers (csrc: gemm_chain_resident_kernel for f16x2, gemm_chain_kernel for bf16x3).
extern "C" int morl_gemm_chain_f32(int fmt, int n_chains, int n_layers, const void* const* act_planes, long long act_plane_stride, const float* act_scale,
                                   const void* const* w_planes, long long w_plane_stride, const float* const* w_scales, const float* const* biases,
                                   int relu, const void* const* relu_bits_in, void* const* relu_bits_out, int M, int K, int k_first, void* stream) {
    using namespace morl;
    MORL_REQUIRE(act_planes && w_planes, MORL_ERR_NULL, "morl_gemm_chain_f32: NULL pointer argument");
    MORL_REQUIRE(n_chains >= 1 && n_chains <= 2 && n_layers >= 1 && n_chains * n_layers <= kChainMaxJobs, MORL_ERR_SHAPE,
                 "morl_gemm_chain_f32: need 1 <= n_chains <= 2 and n_chains * n_layers <= %d (got %d x %d)", kChainMaxJobs, n_chains, n_layers);
    MORL_REQUIRE(morl_gemm_chain_supported(fmt, M, K), MORL_ERR_UNSUPPORTED, "morl_gemm_chain_f32: unsupported configuration fmt=%d M=%d K=%d (256-wide layers, M >= 256)",
                 fmt, M, K);
    // f16x2 runs on the resident kernel (32-wide K blocks), bf16x3 on gemm_chain_kernel
    const int BK = fmt == MORL_FMT_F16X2 ? ResPlan::BK : fmt_bk(fmt);
    if (k_first <= 0) k_first = K;
    MORL_REQUIRE(k_first % BK == 0 && k_first <= K, MORL_ERR_SHAPE, "morl_gemm_chain_f32: k_first=%d must be a multiple of %d and <= K", k_first, BK);
    const uint32_t every_output = (1u << (n_chains * n_layers)) - 1u;
    if (fmt == MORL_FMT_F16X2) {
        ResChainArgs g;
        memset(&g, 0, sizeof(g));
        g.store = every_output;
        const void* in[2] = {nullptr, nullptr};
        for (int c = 0; c < n_chains; ++c) in[c] = act_planes[c * (n_layers + 1)];
        return launch_chain_resident(g, n_chains, n_layers, k_first, in, act_planes, act_plane_stride, act_scale, w_planes, w_plane_stride, w_scales,
                                     biases, relu, relu_bits_in, relu_bits_out, M, K, "morl_gemm_chain_f32", stream);
    }
    ChainMaps maps;  // (host staging of the 3 x 8 tensor maps on this thread's stack -- the entry point stays re-entrant; copied into the kernel
                     // parameters by the launch)
    ChainArgs g;
    memset(&g, 0, sizeof(g));
    const int rc = set_chain_args(g, maps.B, maps.C, fmt, n_chains, n_layers, M, K, k_first, act_planes, act_plane_stride, act_scale, every_output,
                                  w_planes, w_plane_stride, w_scales, biases, relu, relu_bits_in, relu_bits_out, "morl_gemm_chain_f32");
    if (rc) return rc;
    g.n_stages = KPlan<MORL_FMT_BF16X3>::kStages;
    for (int c = 0; c < n_chains; ++c)
        for (int l = 0; l < n_layers; ++l) {
            // the input of job (c, l) is the output of job (c, l - 1); layer 0 may read a narrower input [P][M][k_first] (plane stride M k_first)
            const void* a_in = act_planes[c * (n_layers + 1) + l];
            MORL_REQUIRE(a_in && aligned16(a_in), MORL_ERR_NULL, "morl_gemm_chain_f32: NULL or misaligned input planes (chain %d, layer %d)", c, l);
            const int rca = make_plane_map(&maps.A[c * n_layers + l], fmt, a_in, M, l == 0 ? k_first : K, l == 0 ? (long long)M * k_first : act_plane_stride,
                                           kGemmBM, BK);
            MORL_REQUIRE(rca == 0, MORL_ERR_NO_DEVICE, "morl_gemm_chain_f32: cuTensorMapEncodeTiled(A) failed (%d)", rca);
        }
    const int sms = sm_count();
    const int n_tiles = (M + kGemmBM - 1) / kGemmBM;
    constexpr size_t smem = KPlan<MORL_FMT_BF16X3>::kBytes;
    set_smem_limit_once<gemm_chain_kernel>(smem);
    launch_k_pdl(true, gemm_chain_kernel, dim3(n_tiles < sms ? n_tiles : sms), dim3(kGemmThreads), smem, static_cast<cudaStream_t>(stream), maps, g);
    return check_launch("morl_gemm_chain_f32");
}

// Hidden layers 2.. of one or two pair networks in ONE launch, starting from the separable first layer: the input tile of chain c is
// relu(u[c][b] + v[c][j]) * act_scale (row b W + j, exactly morl_pairs_relu_split_planes' planes) built in shared memory, so the first hidden
// activation never reaches global memory.  Job (c, l) = layer l of chain c; its output planes acts[c n_layers + l] ([P][B W][256]) are written
// only when bit (c n_layers + l) of store_mask is set (NULL otherwise).  f16x2 only (csrc: gemm_chain_resident_kernel).
extern "C" int morl_gemm_chain_pairs_f32(int n_chains, int n_layers, const float* const* u, const float* const* v, int B, int W, const void* const* acts,
                                         long long act_plane_stride, const float* act_scale, const void* const* w_planes, long long w_plane_stride,
                                         const float* const* w_scales, const float* const* biases, void* const* relu_bits_out, unsigned int store_mask,
                                         void* stream) {
    using namespace morl;
    MORL_REQUIRE(u && v && w_planes, MORL_ERR_NULL, "morl_gemm_chain_pairs_f32: NULL pointer argument");
    MORL_REQUIRE(n_chains >= 1 && n_chains <= 2 && n_layers >= 1 && n_chains * n_layers <= kChainMaxJobs, MORL_ERR_SHAPE,
                 "morl_gemm_chain_pairs_f32: need 1 <= n_chains <= 2 and n_chains * n_layers <= %d (got %d x %d)", kChainMaxJobs, n_chains, n_layers);
    MORL_REQUIRE(B > 0 && W > 0 && (long long)B * W <= 0x7fffffffLL && morl_gemm_chain_supported(MORL_FMT_F16X2, B * W, 256), MORL_ERR_SHAPE,
                 "morl_gemm_chain_pairs_f32: bad shape B=%d W=%d (need B W >= 256)", B, W);
    MORL_REQUIRE(store_mask < (1u << (n_chains * n_layers)), MORL_ERR_SHAPE, "morl_gemm_chain_pairs_f32: store_mask 0x%x names jobs beyond %d x %d", store_mask,
                 n_chains, n_layers);
    MORL_REQUIRE(store_mask == 0 || acts, MORL_ERR_NULL, "morl_gemm_chain_pairs_f32: stored outputs need their planes");
    ResChainArgs g;
    memset(&g, 0, sizeof(g));
    g.store = store_mask;
    g.W = W;
    const void* outs[2 * (kChainMaxJobs + 1)] = {};
    for (int c = 0; c < n_chains; ++c) {
        MORL_REQUIRE(u[c] && v[c] && aligned16(u[c]) && aligned16(v[c]), MORL_ERR_ALIGN, "morl_gemm_chain_pairs_f32: u / v of chain %d NULL or not 16-byte aligned", c);
        g.u[c] = u[c];
        g.v[c] = v[c];
        for (int l = 0; l < n_layers; ++l) outs[c * (n_layers + 1) + l + 1] = acts ? acts[c * n_layers + l] : nullptr;
    }
    return launch_chain_resident(g, n_chains, n_layers, 256, nullptr, outs, act_plane_stride, act_scale, w_planes, w_plane_stride, w_scales, biases, 1, nullptr,
                                 relu_bits_out, B * W, 256, "morl_gemm_chain_pairs_f32", stream);
}
