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
    const uint16_t* mask;        // plane 0 of the forward activation [M][ld_mask] for the ReLU-backward mask, or nullptr
    int ld_mask;
    const uint32_t* bits_in;     // ReLU-backward mask as BITS [M][relu_bits_words(N_pad)] words (see morl_b200.h "ReLU bit masks"), or nullptr
    uint32_t* bits_out;          // forward: bit = (output > 0) per column, same layout, or nullptr
    int bits_ld;                 // words per row of bits_in / bits_out: relu_bits_words(N_pad) (the epilogue visits every chunk below N_pad)
    int n_stages;                // depth of the TMA ring: as many (A box + B boxes) stages as fit (2 at N_pad = 256, more for narrow outputs)
    uint32_t b_stage;            // bytes of one B stage slot (the B rows of a stage rounded up to 1 KB)
    int relu;
    const float* a_scale;        // device scalars (powers of two) the A / B planes were scaled by; nullptr = 1
    const float* b_scale;
    const float* c_scale;        // scale applied to the output before it is re-split into c_planes; nullptr = 1
    int l2_hint;                 // L2 eviction hints on the operand loads (MORL_GEMM_L2HINT=1, default off): A evict_first, B evict_last
    int pdl;                     // launched with programmatic stream serialisation: overlap this grid's prologue with the predecessor's tail
    int reverse;                 // walk the row tiles from the last to the first (see morl_gemm_planes_f32: L2 reuse between chained layers)
    unsigned long long* stats;   // diagnostics (MORL_GEMM_STATS=1), else nullptr: [0] consumer wait-on-TMA cycles, [1] consumer loop total,
                                 // [2] producer wait-on-free-stage, [3] epilogue busy
};

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

// One work unit of a consumer warpgroup: D[64 x N] = sum over the K blocks of the staged planes, NPROD products per K step in the order of
// PlaneFmt (small terms first).  A stage goes back to the producer as soon as the MMAs reading it have completed: one group of
// wgmma stays in flight while the next stage is awaited.
// SPLIT = 1 ("split accumulators", N <= 128): the tensor cores accumulate in fp32 with limited-precision alignment at every MMA; with all
// NPROD x K/16 products in one accumulator the rounding of the correction products happens at the magnitude of the running sum.  In split
// mode the LEADING products A0B0 go to acc[0, 64) and the correction products (2^-11 / 2^-8 of the magnitude) to acc[64, 128), so only
// K/16 accumulations happen at full magnitude; the epilogue adds the two with one correctly rounded fp32 add.
template <int FMT, int N, int SPLIT>
__device__ __forceinline__ void mma_unit(float (&acc)[128], uint8_t* smA, uint8_t* smB, uint32_t a_stage_bytes, uint32_t b_stage_stride, int n_kblk,
                                         uint64_t* full, uint64_t* empty, uint32_t& stage, uint32_t& phase, uint32_t n_stages, int wg, int lane,
                                         long long* wait_cycles) {
    using F = PlaneFmt<FMT>;
    static_assert(!SPLIT || N <= 128, "split accumulators: two N / 2-register accumulators per thread");
    constexpr uint32_t ROWB = F::BK * 2;
    constexpr uint32_t a_plane = kGemmBM * ROWB, b_plane = (uint32_t)N * ROWB;
    uint32_t prev = 0;
    for (int kb = 0; kb < n_kblk; ++kb) {
        const long long c0 = wait_cycles ? clock64() : 0;
        g_mbar_wait(&full[stage], phase);
        if (wait_cycles) *wait_cycles += clock64() - c0;
        wgmma_fence();
        const uint32_t a0 = g_smem_u32(smA + stage * a_stage_bytes) + (uint32_t)wg * 64u * ROWB;
        const uint32_t b0 = g_smem_u32(smB + stage * b_stage_stride);
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
            if (lane == 0) g_mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == n_stages) {
            stage = 0;
            phase ^= 1u;
        }
    }
    wgmma_wait<0>();
    if (n_kblk > 0 && lane == 0) g_mbar_arrive(&empty[prev]);
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
    const uint16_t* mask;
    int ld_mask;
    float* c_f32;
    int ldc;
    int planes;                  // re-split the output into planes through tmC
    int ldp;
};

// Epilogue of one 32-column chunk of a consumer warp's 16 accumulator rows [rbase, rbase + 16): thread l holds a[4 q + 2 h + e] = column
// col0 + 8 q + 2 (l % 4) + e of row rbase + l / 4 + 8 h (the wgmma fragment).  The re-split planes leave through the warp's two staging tiles in
// turn (n_stored counts the warp's bulk stores): a chunk is staged while the TMA store of the previous one is still reading the other tile.
template <int FMT>
__device__ __forceinline__ void epilogue_chunk(const float (&a)[16], int col0, int rbase, int lane, const EpiArgs& e, const CUtensorMap* tmC,
                                               uint8_t* my_stage, uint32_t& n_stored, float& amax) {
    using F = PlaneFmt<FMT>;
    constexpr int P = F::P;
    const int l4 = lane & 3, lr = lane >> 2;
    // ReLU bit masks: the word of the row that holds columns [col0, col0 + 32)
    const int wi = relu_bits_word(col0);
    float x[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                float f = __fmaf_rn(a[4 * q + 2 * h + c], e.k_acc, e.bias_s[col0 + 8 * q + 2 * l4 + c]);
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
    if (e.mask) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rbase + lr + 8 * h;
            if (row < e.M) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint32_t mm = __ldg(reinterpret_cast<const uint32_t*>(e.mask + (size_t)row * e.ld_mask + col0 + 8 * q + 2 * l4));
                    // (bf16 or fp16) > 0  <=>  sign bit clear and magnitude non-zero (NaN never occurs in a ReLU output)
                    if ((mm & 0x8000u) || (mm & 0x7FFFu) == 0u) x[h][2 * q] = 0.f;
                    if ((mm & 0x80000000u) || (mm & 0x7FFF0000u) == 0u) x[h][2 * q + 1] = 0.f;
                }
            }
        }
    }
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
        // stage the warp's [16 rows x 32 cols] x P planes in shared memory (TMA SWIZZLE_64B pattern: 16-byte chunk index XOR ((row >> 1) & 3),
        // bank-conflict free), then ONE bulk tensor store writes it out coalesced and asynchronously
        uint8_t* tile = my_stage + (n_stored & 1u) * (uint32_t)(P * 1024);
        ++n_stored;
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // the store before the previous one has read this tile
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rl = lr + 8 * h;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int col = col0 + 8 * q + 2 * l4;
                // ragged last chunk: columns [N, ldp) are written as zero
                const float x0 = col < e.N ? x[h][2 * q] * e.c_mul : 0.f, x1 = col + 1 < e.N ? x[h][2 * q + 1] * e.c_mul : 0.f;
                uint32_t w[P];
                F::split2(x0, x1, w, amax);  // re-split (c_scale x) into P planes, two columns per word
                uint8_t* st = tile + rl * 64 + ((q ^ ((rl >> 1) & 3)) << 4) + 4 * l4;
#pragma unroll
                for (int p = 0; p < P; ++p) *reinterpret_cast<uint32_t*>(st + p * 1024) = w[p];
            }
        }
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

// One CTA per 128-row tile.  SPLIT = 1: see mma_unit; a tile wider than 128 columns is then computed as column units of 128 (the A boxes of
// the tile are staged once per unit).  SPLIT = 0 and N_pad > 256: two column units [0, 256) and [256, N_pad), each with the stage plan of
// N_pad = 256 and this unit's 256 biases in shared memory.
template <int FMT, int SPLIT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_planes_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                   const GemmArgs g) {
    using F = PlaneFmt<FMT>;
    using L = KPlan<FMT>;
    constexpr int P = F::P;
    constexpr int BK = F::BK;
    constexpr int kMaxStages = L::kMaxStages;
    constexpr uint32_t ROWB = L::kRowB;
    const uint32_t kStages = (uint32_t)g.n_stages;  // runtime: narrow outputs leave room for a deeper ring (host: morl_gemm_planes_f32)
    extern __shared__ uint8_t gsmem_raw[];
    // 1 KB alignment by pointer arithmetic ON the shared array (not through an integer cast), so that the compiler keeps every derived
    // pointer in the shared address space: through the cast the bias / staging accesses were generic LD.E / ST.E (long-scoreboard stalls)
    uint8_t* gsmem = gsmem_raw + ((1024u - (g_smem_u32(gsmem_raw) & 1023u)) & 1023u);
    const int BN = g.N_pad;
    constexpr uint32_t a_stage_bytes = L::kAStage;
    const uint32_t b_stage_stride = g.b_stage;
    uint8_t* smA = gsmem;
    uint8_t* smB = gsmem + kStages * a_stage_bytes;  // (n_stages * (A + B) <= kOffC, checked on the host)
    uint8_t* stage_c = gsmem + L::kOffC;  // per-consumer-warp staging tiles for the TMA store of the re-split activations
    uint64_t* full = reinterpret_cast<uint64_t*>(gsmem + L::kOffBar);
    uint64_t* empty = full + kMaxStages;
    float* bias_s = reinterpret_cast<float*>(gsmem + L::kOffBias);  // [256]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_tiles = (g.M + kGemmBM - 1) / kGemmBM;
    const int n_kblk = g.K / BK;
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
        for (uint32_t s = 0; s < kStages; ++s) {
            g_mbar_init(&full[s], 1);
            g_mbar_init(&empty[s], 8);  // one arrival per consumer warp
        }
        g_mbar_init_fence();
    }
    if (g.pdl) {
        // programmatic dependent launch: this grid may have become resident (barrier init above) while the previous kernel
        // of the stream was still draining its last tiles; let OUR successor do the same, then wait until the predecessor's results are
        // visible -- nothing above this line reads global memory, everything below may
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    for (int t = threadIdx.x; t < 256; t += blockDim.x) bias_s[t] = (g.bias && t < g.N) ? g.bias[t] : 0.f;
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: one lane issues TMA =================
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
            uint32_t stage = 0, phase = 0;
            long long w_empty = 0;
            const uint64_t pol_a = l2_policy_evict_first(), pol_b = l2_policy_evict_last();
            for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
                int tile, n_begin, n_cnt;
                unit_of(u, tile, n_begin, n_cnt);
                const int row0 = tile * kGemmBM;
                const uint32_t b_plane = (uint32_t)n_cnt * ROWB;
                for (int kb = 0; kb < n_kblk; ++kb) {
                    const long long c0 = g.stats ? clock64() : 0;
                    g_mbar_wait(&empty[stage], phase ^ 1u);
                    if (g.stats) w_empty += clock64() - c0;
                    g_mbar_expect_tx(&full[stage], a_stage_bytes + (uint32_t)P * b_plane);
                    uint8_t* bs = smB + stage * b_stage_stride;
                    if (g.l2_hint) tma_load_3d_hint(smA + stage * a_stage_bytes, &tmA, &full[stage], kb * BK, row0, 0, pol_a);
                    else tma_load_3d(smA + stage * a_stage_bytes, &tmA, &full[stage], kb * BK, row0, 0);
                    for (int p = 0; p < P; ++p)
                        for (int r = 0; r < n_cnt; r += kGemmBoxN) {
                            uint8_t* dst = bs + (uint32_t)p * b_plane + (uint32_t)r * ROWB;
                            if (g.l2_hint) tma_load_3d_hint(dst, &tmB, &full[stage], kb * BK, n_begin + r, p, pol_b);
                            else tma_load_3d(dst, &tmB, &full[stage], kb * BK, n_begin + r, p);
                        }
                    if (++stage == kStages) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
            if (g.stats) atomicAdd(&g.stats[2], (unsigned long long)w_empty);
        }
    } else {
        // ================= consumer warpgroups (warps 0..7) =================
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2;
        uint8_t* my_stage = stage_c + warp * 2 * L::kStageC;
        uint32_t n_stored = 0;
        // x = acc / (sA sB) + bias; when only planes are written (the hidden layers) the output scale is FOLDED into the two constants:
        // fold * x = acc * (fold / (sA sB)) + fold * bias (exact, powers of two), and max / mask commute with a positive factor
        const float c_mul = ld_scale(g.c_scale);
        const bool folded = g.c_f32 == nullptr;
        const float fold = folded ? c_mul : 1.0f;
        if (warp == 0 && folded)  // (bias_s was filled before the CTA barrier; one warp rescales it)
            for (int t = lane; t < 256; t += 32) bias_s[t] *= fold;
        asm volatile("bar.sync 1, 256;" ::: "memory");  // the 8 consumer warps only
        EpiArgs e;
        e.M = g.M; e.N = g.N;
        e.k_acc = fold / (ld_scale(g.a_scale) * ld_scale(g.b_scale));
        e.c_mul = folded ? 1.0f : c_mul;
        e.bias_s = bias_s; e.relu = g.relu; e.bits_in = g.bits_in; e.bits_out = g.bits_out; e.bits_ld = g.bits_ld; e.mask = g.mask;
        e.ld_mask = g.ld_mask; e.c_f32 = g.c_f32; e.ldc = g.ldc; e.planes = g.c_planes != nullptr; e.ldp = g.ldp;
        float amax = 0.f;
        float acc[128];
        uint32_t stage = 0, phase = 0;
        long long w_full = 0, busy = 0;
        long long* wc = g.stats ? &w_full : nullptr;
        const long long t_begin = g.stats ? clock64() : 0;
        for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
            int tile, n_begin, n_cnt;
            unit_of(u, tile, n_begin, n_cnt);
#define MORL_UNIT(N_) \
    case N_: mma_unit<FMT, N_, SPLIT>(acc, smA, smB, a_stage_bytes, b_stage_stride, n_kblk, full, empty, stage, phase, kStages, wg, lane, wc); break;
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
            const long long c1 = g.stats ? clock64() : 0;
            if (wide) {
                // this unit's biases (times the folded output scale), indexed by output column: every consumer warp has left the previous
                // unit's epilogue (both warpgroups have finished the MMAs of this unit)
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const int col = n_begin + (int)threadIdx.x;
                bias_s[threadIdx.x] = (g.bias && col < g.N) ? g.bias[col] * fold : 0.f;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                e.bias_s = bias_s - n_begin;
            }
            const int rbase = tile * kGemmBM + wg * 64 + (warp & 3) * 16;
#pragma unroll
            for (int c = 0; c < (SPLIT ? 4 : 8); ++c) {
                if (32 * c < n_cnt) {
                    float a[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) a[j] = SPLIT ? __fadd_rn(acc[16 * c + j], acc[64 + 16 * c + j]) : acc[16 * c + j];
                    epilogue_chunk<FMT>(a, n_begin + 32 * c, rbase, lane, e, &tmC, my_stage, n_stored, amax);
                }
            }
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
// CHAIN kernel: several dense hidden layers of one or two networks in ONE persistent launch (f16x2 / bf16x3 planes, N = 256 wide
// layers).  A layer's output rows depend only on the same rows of its input, so a CTA can take one of its 128-row tiles through ALL
// layers: the tile it stores for layer l is the tile it loads for layer l+1 a few units later -- by then still in the 50 MB L2, so only the
// first layer's input is read from HBM, and the launch prologue / drain is paid once instead of per layer.  Work of a CTA: its tiles in
// groups of `lanes / n_chains`; per group, for every layer, one unit per LANE (lane = (chain, tile
// of the group)): four lanes keep the dependency distance at four units (unit (l, lane) needs the stores of unit (l-1, lane)), so the
// producer never waits for the epilogue that has just finished.  Same roles, barriers and arithmetic as gemm_planes_kernel<FMT, 0>
// (bit-identical outputs: tests/test_gemm_gpu.py); additional barrier stored[lane]: the consumer warps arrive once their bulk
// stores of the unit have COMPLETED, the producer waits for it before loading the next layer of that lane.
// =================================================================================================================
constexpr int kChainMaxJobs = 8;   // chains x layers
constexpr int kChainLanes = 4;

struct alignas(64) ChainMaps {
    CUtensorMap A[kChainMaxJobs];  // load map of the INPUT of job (chain c, layer l): [P][M][K], box P x 128 x BK
    CUtensorMap B[kChainMaxJobs];  // weight planes of the job: [P][256][K], box 1 x 32 x BK
    CUtensorMap C[kChainMaxJobs];  // store map of the OUTPUT of the job: [P][M][256], box P x 16 x 32 (64-byte swizzle)
};

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
    int n_stages;
    int pdl;
};

template <int FMT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_chain_kernel(const __grid_constant__ ChainMaps maps, const ChainArgs g) {
    using F = PlaneFmt<FMT>;
    using L = KPlan<FMT>;
    constexpr int P = F::P;
    constexpr int BK = F::BK;
    constexpr int BN = 256;
    constexpr int kMaxStages = L::kMaxStages;
    constexpr uint32_t ROWB = L::kRowB;
    const uint32_t kStages = (uint32_t)g.n_stages;
    extern __shared__ uint8_t gsmem_raw[];
    uint8_t* gsmem = gsmem_raw + ((1024u - (g_smem_u32(gsmem_raw) & 1023u)) & 1023u);
    constexpr uint32_t a_stage_bytes = L::kAStage;
    constexpr uint32_t b_stage_bytes = L::kBStage;
    uint8_t* smA = gsmem;
    uint8_t* smB = gsmem + kStages * a_stage_bytes;
    uint8_t* stage_c = gsmem + L::kOffC;
    uint64_t* full = reinterpret_cast<uint64_t*>(gsmem + L::kOffBar);
    uint64_t* empty = full + kMaxStages;
    uint64_t* stored = empty + kMaxStages;  // [kChainLanes]
    float* bias_s = reinterpret_cast<float*>(gsmem + L::kOffBias);  // [256], refilled per unit by the consumer warps

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int unit = blockIdx.x, n_units = gridDim.x;
    const int n_tiles = (g.M + kGemmBM - 1) / kGemmBM;
    const int n_kblk_full = g.K / BK, n_kblk_first = g.k_first / BK;
    const int tiles_per_group = kChainLanes / g.n_chains;  // lanes of a group: (tile of the group) x (chain)
    // Tile t of chain c goes to CTA (t + offset_c) mod n_units with a DIFFERENT rotation per chain: when the tiles do not divide evenly, both
    // chains on the same CTAs would give some CTAs two extra tiles and others none; rotated by half the grid the remainders spread.
    const int cu0 = unit, cu1 = (unit + n_units / 2) % n_units;
    const int mt0 = cu0 < n_tiles ? (n_tiles - cu0 + n_units - 1) / n_units : 0;
    const int mt1 = g.n_chains > 1 ? (cu1 < n_tiles ? (n_tiles - cu1 + n_units - 1) / n_units : 0) : 0;
    const int n_groups = ((mt0 > mt1 ? mt0 : mt1) + tiles_per_group - 1) / tiles_per_group;
    // unit (group gi, layer l, lane ln) -> (job, tile) or tile = -1 (no such tile for this CTA)
    auto unit_of = [&](int gi, int l, int ln, int& job, int& tile) {
        const int c = ln % g.n_chains, ti = gi * tiles_per_group + ln / g.n_chains;
        job = c * g.n_layers + l;
        tile = ti < (c ? mt1 : mt0) ? (c ? cu1 : cu0) + ti * n_units : -1;
    };

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) {
            g_mbar_init(&full[s], 1);
            g_mbar_init(&empty[s], 8);
        }
        for (int s = 0; s < kChainLanes; ++s) g_mbar_init(&stored[s], 8);  // the 8 consumer warps
        g_mbar_init_fence();
    }
    if (g.pdl) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: one lane issues TMA =================
        warpgroup_reg_dec<kGemmProducerRegs>();
        if (warp == 8 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            uint32_t done_on_lane[kChainLanes] = {0u, 0u, 0u, 0u};  // units already issued on each lane = completions of stored[lane] to expect
            for (int gi = 0; gi < n_groups; ++gi)
                for (int l = 0; l < g.n_layers; ++l)
                    for (int ln = 0; ln < kChainLanes; ++ln) {
                        int job, tile;
                        unit_of(gi, l, ln, job, tile);
                        if (tile < 0) continue;
                        if (l > 0) {
                            // the input tile of this unit is the output tile of the lane's previous unit: wait until the stores of
                            // it have completed (completion number done_on_lane[ln] of stored[ln])
                            g_mbar_wait(&stored[ln], (done_on_lane[ln] - 1u) & 1u);
                            asm volatile("fence.proxy.async.global;" ::: "memory");
                        }
                        ++done_on_lane[ln];
                        const int row0 = tile * kGemmBM;
                        const int n_kblk = l == 0 ? n_kblk_first : n_kblk_full;
                        for (int kb = 0; kb < n_kblk; ++kb) {
                            g_mbar_wait(&empty[stage], phase ^ 1u);
                            g_mbar_expect_tx(&full[stage], a_stage_bytes + b_stage_bytes);
                            tma_load_3d(smA + stage * a_stage_bytes, &maps.A[job], &full[stage], kb * BK, row0, 0);
                            for (int p = 0; p < P; ++p)
                                for (int r = 0; r < BN; r += kGemmBoxN)
                                    tma_load_3d(smB + stage * b_stage_bytes + (uint32_t)(p * BN + r) * ROWB, &maps.B[job], &full[stage], kb * BK, r, p);
                            if (++stage == kStages) {
                                stage = 0;
                                phase ^= 1u;
                            }
                        }
                    }
        }
    } else {
        // ================= consumer warpgroups (warps 0..7) =================
        warpgroup_reg_inc<kGemmConsumerRegs>();
        const int wg = warp >> 2;
        uint8_t* my_stage = stage_c + warp * 2 * L::kStageC;
        uint32_t n_stored = 0;
        const float s_act = ld_scale(g.a_scale);
        float amax = 0.f;
        float acc[128];
        uint32_t stage = 0, phase = 0;
        for (int gi = 0; gi < n_groups; ++gi)
            for (int l = 0; l < g.n_layers; ++l)
                for (int ln = 0; ln < kChainLanes; ++ln) {
                    int job, tile;
                    unit_of(gi, l, ln, job, tile);
                    if (tile < 0) continue;
                    // this unit's bias (times the folded output scale) into shared memory: every consumer warp has left the previous unit
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    bias_s[threadIdx.x] = (g.bias[job] ? __ldg(g.bias[job] + threadIdx.x) : 0.f) * s_act;
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    EpiArgs e;
                    e.M = g.M; e.N = BN;
                    // x * s_act = acc * (s_act / (s_act * sB)) + s_act * bias  (powers of two: exact), as gemm_planes_kernel's folded epilogue
                    e.k_acc = s_act / (s_act * ld_scale(g.b_scale[job]));
                    e.c_mul = 1.0f;
                    e.bias_s = bias_s; e.relu = g.relu; e.bits_in = g.bits_in[job]; e.bits_out = g.bits_out[job]; e.bits_ld = relu_bits_words(BN);
                    e.mask = nullptr; e.ld_mask = 0;
                    e.c_f32 = nullptr; e.ldc = 0; e.planes = 1; e.ldp = BN;
                    mma_unit<FMT, BN, 0>(acc, smA, smB, a_stage_bytes, b_stage_bytes, l == 0 ? n_kblk_first : n_kblk_full, full, empty, stage, phase, kStages,
                                         wg, lane, nullptr);
                    const int rbase = tile * kGemmBM + wg * 64 + (warp & 3) * 16;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        float a[16];
#pragma unroll
                        for (int j = 0; j < 16; ++j) a[j] = acc[16 * c + j];
                        epilogue_chunk<FMT>(a, 32 * c, rbase, lane, e, &maps.C[job], my_stage, n_stored, amax);
                    }
                    // the lane's next layer loads what this unit stored (bit masks included): signal once the bulk stores of this warp have completed
                    __syncwarp();
                    if (lane == 0) {
                        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
                        g_mbar_arrive(&stored[ln]);
                    }
                }
        if (FMT == MORL_FMT_F16X2) note_overflow(amax);
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
    // 1 KB alignment by pointer arithmetic ON the shared array (not through an integer cast), so that the compiler keeps every derived
    // pointer in the shared address space: through the cast the bias / staging accesses were generic LD.E / ST.E (long-scoreboard stalls)
    uint8_t* gsmem = gsmem_raw + ((1024u - (g_smem_u32(gsmem_raw) & 1023u)) & 1023u);
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
    uint32_t* ones = reinterpret_cast<uint32_t*>(ones_b + ((1024u - (g_smem_u32(ones_b) & 1023u)) & 1023u));
    for (int t = threadIdx.x; t < 1024; t += blockDim.x) ones[t] = F::kOnes2;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nt = blockIdx.x % g.n_tiles;
    const int split = blockIdx.x / (g.n_tiles * k_units);
    const int m_begin = split * g.rows_per_split;
    const int m_end = min(g.M, m_begin + g.rows_per_split);
    const int n_kblk = (m_end - m_begin + kMnKT - 1) / kMnKT;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            g_mbar_init(&full[s], 1);
            g_mbar_init(&empty[s], 8);  // one arrival per consumer warp
        }
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
template <int FMT>
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
        const float x[8] = {u0.x + v0.x, u0.y + v0.y, u0.z + v0.z, u0.w + v0.w, u1.x + v1.x, u1.y + v1.y, u1.z + v1.z, u1.w + v1.w};
        uint32_t o[F::P][4];
        uint32_t pos = 0;  // bit t = (column 8 h8 + t is positive)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint32_t w[F::P];
            const float r0 = x[2 * q] < 0.f ? 0.f : x[2 * q], r1 = x[2 * q + 1] < 0.f ? 0.f : x[2 * q + 1];  // NaN-propagating ReLU
            pos |= (r0 > 0.f ? 1u : 0u) << (2 * q) | (r1 > 0.f ? 1u : 0u) << (2 * q + 1);
            F::split2(r0 * s, r1 * s, w, amax);
#pragma unroll
            for (int p = 0; p < F::P; ++p) o[p][q] = w[p];
        }
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
            uint32_t pos = 0;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                uint32_t w[F::P];
                const float r0 = x[2 * t] < 0.f ? 0.f : x[2 * t], r1 = x[2 * t + 1] < 0.f ? 0.f : x[2 * t + 1];  // NaN-propagating ReLU
                pos |= (r0 > 0.f ? 1u : 0u) << (2 * t) | (r1 > 0.f ? 1u : 0u) << (2 * t + 1);
                F::split2(r0 * s, r1 * s, w, amax);
#pragma unroll
                for (int p = 0; p < F::P; ++p) o[p][t] = w[p];
            }
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
    const int n = morl_device_sm_count();
    return n > 0 && n <= 256 ? n : 132;
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
        static bool attr_set = false;
        if (!attr_set) {
            cudaFuncSetAttribute(gemm_planes_mn_kernel<kFmt>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            attr_set = true;
        }
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

extern "C" int morl_colsum_planes(int fmt, const void* planes, long long plane_stride, const float* scale, int M, int ld, int N, float* out,
                                  void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_colsum_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(planes && out && workspace, MORL_ERR_NULL, "morl_colsum_planes: NULL pointer argument");
    MORL_REQUIRE(M > 0 && N > 0 && ld >= N && ld % 8 == 0 && plane_stride % 8 == 0, MORL_ERR_SHAPE, "morl_colsum_planes: bad shape M=%d N=%d ld=%d", M, N, ld);
    const int chunks = 296;
    const int rpc = (M + chunks - 1) / chunks;
    const int nch = (M + rpc - 1) / rpc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* part = static_cast<float*>(workspace);
    MORL_DISPATCH_FMT(fmt, (colsum_planes_kernel<kFmt><<<dim3((unsigned)nch, (unsigned)((ld + 255) / 256)), dim3(32, 8), 0, st>>>(
                               static_cast<const uint16_t*>(planes), plane_stride, M, ld, N, rpc, part)));
    int rc = check_launch("morl_colsum_planes");
    if (rc) return rc;
    launch_k(reduce_partials_kernel, dim3((N + 31) / 32), dim3(dim3(32, 8)), 0, st, part, nch, 1, N, 1, N, 0, out, N, 1 << 30, nullptr, nullptr, scale, nullptr);
    return check_launch("morl_colsum_planes(reduce)");
}

extern "C" int morl_pairs_grad_reduce_planes(int fmt, const void* planes, long long plane_stride, const float* scale, int B, int W, int H, float* dU,
                                             float* dV, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_pairs_grad_reduce_planes: unknown plane format %d", fmt);
    MORL_REQUIRE(planes && dU && dV && workspace, MORL_ERR_NULL, "morl_pairs_grad_reduce_planes: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && H > 0 && H % 8 == 0 && plane_stride % 8 == 0, MORL_ERR_SHAPE, "morl_pairs_grad_reduce_planes: bad shape B=%d W=%d H=%d", B, W, H);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint16_t* pl = static_cast<const uint16_t*>(planes);
    if (W <= 64) {
        // one pass: dU directly, dV as per-chunk partials [chunks][W*H] reduced in a fixed order
        int bpc = (B + 295) / 296;  // <= 296 chunks (the documented workspace size), at most kPgrMaxB transitions per chunk
        if (bpc > kPgrMaxB) bpc = kPgrMaxB;
        const int nchf = (B + bpc - 1) / bpc;
        if (nchf <= 296) {
            const int Nf = W * H;
            float* partf = static_cast<float*>(workspace);
            const size_t smemf = (size_t)kPgrMaxB * 8 * 32 * 9 * sizeof(float);  // 73,728 B
            MORL_DISPATCH_FMT(fmt, {
                static bool configured = false;
                if (!configured) {
                    cudaFuncSetAttribute(pairs_grad_reduce_fused_kernel<kFmt>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemf);
                    configured = true;
                }
                launch_k(pairs_grad_reduce_fused_kernel<kFmt>, dim3(dim3((unsigned)nchf, (unsigned)((H + 255) / 256))), dim3(dim3(32, 8)), smemf, st, pl, plane_stride, B, W,
                                                                                                                                     H, bpc, dU, partf, scale);
            });
            int rcf = check_launch("morl_pairs_grad_reduce_planes(fused)");
            if (rcf) return rcf;
            launch_k(reduce_partials_kernel, dim3((Nf + 31) / 32), dim3(dim3(32, 8)), 0, st, partf, nchf, 1, Nf, 1, Nf, 0, dV, Nf, 1 << 30, nullptr, nullptr, scale, nullptr);
            return check_launch("morl_pairs_grad_reduce_planes(reduce)");
        }
    }
    // dU[b] = sum over the W rows of transition b
    MORL_DISPATCH_FMT(fmt, (pairs_rowblock_sum_kernel<kFmt><<<dim3((unsigned)B, (unsigned)((H + 255) / 256)), dim3(32, 8), 0, st>>>(pl, plane_stride, W, H,
                                                                                                                                     dU, scale)));
    int rc = check_launch("morl_pairs_grad_reduce_planes(dU)");
    if (rc) return rc;
    // dV[j] = sum over b: column sums of the [B, W*H] view
    const int N = W * H;
    const int chunks = 74;
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
template <int FMT, int SPLIT>
static int launch_gemm_planes(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmArgs& g, int sms, cudaStream_t st) {
    constexpr size_t smem = KPlan<FMT>::kBytes;
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(gemm_planes_kernel<FMT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_set = true;
    }
    constexpr int kUnitN = SPLIT ? 128 : 256;  // column units per tile: as gemm_planes_kernel
    const int n_work = (g.M + kGemmBM - 1) / kGemmBM * ((g.N_pad + kUnitN - 1) / kUnitN);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(n_work < sms ? n_work : sms);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g.pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, gemm_planes_kernel<FMT, SPLIT>, tmA, tmB, tmC, g);
    return check_launch("morl_gemm_planes_f32");
}
}  // namespace morl

extern "C" int morl_gemm_planes_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                                    long long b_plane_stride, const float* b_scale, int M, int N, int N_pad, int K, const float* bias, int relu,
                                    const void* relu_mask_plane0, int ld_mask, float* c_f32, int ldc, void* c_planes, int ldp, long long c_plane_stride,
                                    const float* c_scale, int reverse_tiles, int split_accumulators, const void* relu_bits_in, void* relu_bits_out,
                                    void* stream) {
    using namespace morl;
    MORL_REQUIRE(fmt_ok(fmt), MORL_ERR_UNSUPPORTED, "morl_gemm_planes_f32: unknown plane format %d", fmt);
    MORL_REQUIRE(a_planes && b_planes && (c_f32 || c_planes), MORL_ERR_NULL, "morl_gemm_planes_f32: NULL pointer argument");
    MORL_REQUIRE(M > 0 && N > 0 && K > 0 && N_pad >= N, MORL_ERR_SHAPE, "morl_gemm_planes_f32: bad shape M=%d N=%d N_pad=%d K=%d", M, N, N_pad, K);
    const int BK = fmt == MORL_FMT_F16X2 ? PlaneFmt<MORL_FMT_F16X2>::BK : PlaneFmt<MORL_FMT_BF16X3>::BK;
    MORL_REQUIRE(K % BK == 0 && N_pad % 32 == 0 && N_pad <= 512, MORL_ERR_UNSUPPORTED,
                 "morl_gemm_planes_f32: need K %% %d == 0, N_pad %% 32 == 0, N_pad <= 512 (K=%d N_pad=%d)", BK, K, N_pad);
    MORL_REQUIRE(aligned16(a_planes) && aligned16(b_planes), MORL_ERR_ALIGN, "morl_gemm_planes_f32: operand planes must be 16-byte aligned");
    MORL_REQUIRE(aligned16(relu_bits_in) && aligned16(relu_bits_out), MORL_ERR_ALIGN, "morl_gemm_planes_f32: ReLU bit masks must be 16-byte aligned");
    if (c_planes)
        MORL_REQUIRE(ldp % 32 == 0 && ldp >= N && ldp <= N_pad && aligned16(c_planes) && c_plane_stride % 8 == 0, MORL_ERR_SHAPE,
                     "morl_gemm_planes_f32: ldp=%d must be a multiple of 32 with N <= ldp <= N_pad", ldp);
    int sms = morl_device_sm_count();
    if (sms <= 0) sms = 132;
    CUtensorMap tmA, tmB;
    int rc = make_plane_map(&tmA, fmt, a_planes, M, K, a_plane_stride, kGemmBM, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_planes_f32: cuTensorMapEncodeTiled(A) failed (%d)", rc);
    rc = make_plane_map(&tmB, fmt, b_planes, N_pad, K, b_plane_stride, kGemmBoxN, BK, true);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_planes_f32: cuTensorMapEncodeTiled(B) failed (%d)", rc);
    CUtensorMap tmC;
    memset(&tmC, 0, sizeof(tmC));
    if (c_planes) {  // store map of the re-split output: [P][M][ldp], box 32 cols x 16 rows x P planes (64-byte swizzle)
        rc = make_plane_map(&tmC, fmt, c_planes, M, ldp, c_plane_stride, 16, 32);
        MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_planes_f32: cuTensorMapEncodeTiled(C) failed (%d)", rc);
    }
    GemmArgs g;
    g.M = M; g.N = N; g.N_pad = N_pad; g.K = K;
    g.bias = bias; g.c_f32 = c_f32; g.ldc = ldc;
    g.c_planes = c_planes; g.ldp = ldp; g.plane_stride = c_plane_stride;
    g.mask = static_cast<const uint16_t*>(relu_mask_plane0); g.ld_mask = ld_mask; g.relu = relu;
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
        static const int st_env = [] { const char* e = getenv("MORL_GEMM_STAGES"); return e ? atoi(e) : 0; }();
        if (st_env > 0 && st_env < n_st) n_st = st_env;  // A/B measurements
        g.n_stages = n_st;
        g.b_stage = b_box;
    }
    g.a_scale = a_scale; g.b_scale = b_scale; g.c_scale = c_scale;
    g.reverse = reverse_tiles ? 1 : 0;
    // programmatic dependent launch between consecutive GEMMs of a chain (MORL_GEMM_PDL=0 disables it)
    static const bool want_pdl = [] { const char* e = getenv("MORL_GEMM_PDL"); return !(e && e[0] == '0'); }();
    g.pdl = want_pdl ? 1 : 0;
    // L2 eviction hints on the operand loads are opt-in (MORL_GEMM_L2HINT=1)
    static const bool want_hint = [] { const char* e = getenv("MORL_GEMM_L2HINT"); return e && e[0] == '1'; }();
    g.l2_hint = want_hint ? 1 : 0;
    static const bool want_stats = [] { const char* e = getenv("MORL_GEMM_STATS"); return e && e[0] == '1'; }();
    g.stats = nullptr;
    if (want_stats) {
        void* sp = nullptr;
        cudaGetSymbolAddress(&sp, g_gemm_stats);
        g.stats = static_cast<unsigned long long*>(sp);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // accumulator mode (see gemm_planes_kernel): per call; MORL_GEMM_SPLIT_ACC=0 / 1 overrides every call (A/B measurements)
    static const int split_env = [] { const char* e = getenv("MORL_GEMM_SPLIT_ACC"); return e ? (e[0] == '0' ? 0 : 1) : -1; }();
    const bool split_acc = split_env >= 0 ? split_env != 0 : split_accumulators != 0;
    if (fmt == MORL_FMT_F16X2)
        return split_acc ? launch_gemm_planes<MORL_FMT_F16X2, 1>(tmA, tmB, tmC, g, sms, st) : launch_gemm_planes<MORL_FMT_F16X2, 0>(tmA, tmB, tmC, g, sms, st);
    return split_acc ? launch_gemm_planes<MORL_FMT_BF16X3, 1>(tmA, tmB, tmC, g, sms, st) : launch_gemm_planes<MORL_FMT_BF16X3, 0>(tmA, tmB, tmC, g, sms, st);
}


extern "C" int morl_gemm_chain_supported(int fmt, int M, int K) {
    using namespace morl;
    return fmt_ok(fmt) && M >= 2 * kGemmBM && K == 256;
}

// Several 256-wide hidden layers (Linear + ReLU, planes in / planes out) of one or two networks in ONE persistent launch: job (c, l) computes
// act[c][l+1] = relu(act[c][l] . W[c][l]^T + bias[c][l]) exactly as morl_gemm_planes_f32 does (bit-identical), but a CTA takes its row tiles
// through all layers, so intermediate activations are re-read from L2 instead of HBM (csrc: gemm_chain_kernel).
extern "C" int morl_gemm_chain_f32(int fmt, int n_chains, int n_layers, const void* const* act_planes, long long act_plane_stride, const float* act_scale,
                                   const void* const* w_planes, long long w_plane_stride, const float* const* w_scales, const float* const* biases,
                                   int relu, const void* const* relu_bits_in, void* const* relu_bits_out, int M, int K, int k_first, void* stream) {
    using namespace morl;
    MORL_REQUIRE(act_planes && w_planes, MORL_ERR_NULL, "morl_gemm_chain_f32: NULL pointer argument");
    MORL_REQUIRE(n_chains >= 1 && n_chains <= 2 && n_layers >= 1 && n_chains * n_layers <= kChainMaxJobs, MORL_ERR_SHAPE,
                 "morl_gemm_chain_f32: need 1 <= n_chains <= 2 and n_chains * n_layers <= %d (got %d x %d)", kChainMaxJobs, n_chains, n_layers);
    MORL_REQUIRE(morl_gemm_chain_supported(fmt, M, K), MORL_ERR_UNSUPPORTED, "morl_gemm_chain_f32: unsupported configuration fmt=%d M=%d K=%d (256-wide layers, M >= 256)",
                 fmt, M, K);
    const int BK = fmt == MORL_FMT_F16X2 ? PlaneFmt<MORL_FMT_F16X2>::BK : PlaneFmt<MORL_FMT_BF16X3>::BK;
    if (k_first <= 0) k_first = K;
    MORL_REQUIRE(k_first % BK == 0 && k_first <= K, MORL_ERR_SHAPE, "morl_gemm_chain_f32: k_first=%d must be a multiple of %d and <= K", k_first, BK);
    ChainMaps maps;  // (host staging of the 3 x 8 tensor maps on this thread's stack -- the entry point stays re-entrant; copied into the kernel
                     // parameters by the launch)
    ChainArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.K = K; g.k_first = k_first; g.n_chains = n_chains; g.n_layers = n_layers; g.a_scale = act_scale; g.relu = relu ? 1 : 0;
    for (int c = 0; c < n_chains; ++c)
        for (int l = 0; l < n_layers; ++l) {
            const int job = c * n_layers + l;
            const void* a_in = act_planes[c * (n_layers + 1) + l];
            const void* a_out = act_planes[c * (n_layers + 1) + l + 1];
            MORL_REQUIRE(a_in && a_out && w_planes[job] && aligned16(a_in) && aligned16(a_out) && aligned16(w_planes[job]), MORL_ERR_NULL,
                         "morl_gemm_chain_f32: NULL or misaligned plane pointer (chain %d, layer %d)", c, l);
            // layer 0 may read a narrower input [P][M][k_first] (plane stride M * k_first) through weights [P][256][k_first]
            const int kj = l == 0 ? k_first : K;
            const long long a_stride = l == 0 ? (long long)M * k_first : act_plane_stride;
            const long long w_stride = l == 0 ? (long long)256 * k_first : w_plane_stride;
            int rc = make_plane_map(&maps.A[job], fmt, a_in, M, kj, a_stride, kGemmBM, BK);
            MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_chain_f32: cuTensorMapEncodeTiled(A) failed (%d)", rc);
            rc = make_plane_map(&maps.B[job], fmt, w_planes[job], 256, kj, w_stride, kGemmBoxN, BK, true);
            MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_chain_f32: cuTensorMapEncodeTiled(B) failed (%d)", rc);
            rc = make_plane_map(&maps.C[job], fmt, a_out, M, 256, act_plane_stride, 16, 32);
            MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_gemm_chain_f32: cuTensorMapEncodeTiled(C) failed (%d)", rc);
            g.bias[job] = biases ? biases[job] : nullptr;
            g.b_scale[job] = w_scales ? w_scales[job] : nullptr;
            g.bits_out[job] = relu_bits_out ? static_cast<uint32_t*>(relu_bits_out[job]) : nullptr;
            g.bits_in[job] = relu_bits_in ? static_cast<const uint32_t*>(relu_bits_in[job]) : nullptr;
            MORL_REQUIRE(aligned16(g.bits_out[job]) && aligned16(g.bits_in[job]), MORL_ERR_ALIGN, "morl_gemm_chain_f32: ReLU bit masks must be 16-byte aligned");
        }
    g.n_stages = fmt == MORL_FMT_F16X2 ? KPlan<MORL_FMT_F16X2>::kStages : KPlan<MORL_FMT_BF16X3>::kStages;
    static const bool want_pdl = [] { const char* e = getenv("MORL_GEMM_PDL"); return !(e && e[0] == '0'); }();
    g.pdl = want_pdl ? 1 : 0;
    int sms = morl_device_sm_count();
    if (sms <= 0) sms = 132;
    const int n_tiles = (M + kGemmBM - 1) / kGemmBM;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(n_tiles < sms ? n_tiles : sms);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g.pdl ? 1 : 0;
    if (fmt == MORL_FMT_F16X2) {
        constexpr size_t smem = KPlan<MORL_FMT_F16X2>::kBytes;
        static bool attr_set = false;
        if (!attr_set) {
            cudaFuncSetAttribute(gemm_chain_kernel<MORL_FMT_F16X2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            attr_set = true;
        }
        cfg.dynamicSmemBytes = smem;
        cudaLaunchKernelEx(&cfg, gemm_chain_kernel<MORL_FMT_F16X2>, maps, g);
    } else {
        constexpr size_t smem = KPlan<MORL_FMT_BF16X3>::kBytes;
        static bool attr_set = false;
        if (!attr_set) {
            cudaFuncSetAttribute(gemm_chain_kernel<MORL_FMT_BF16X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            attr_set = true;
        }
        cfg.dynamicSmemBytes = smem;
        cudaLaunchKernelEx(&cfg, gemm_chain_kernel<MORL_FMT_BF16X3>, maps, g);
    }
    return check_launch("morl_gemm_chain_f32");
}
