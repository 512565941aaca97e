// gemm_tc.cuh -- wgmma / TMA / mbarrier PTX wrappers, the split-operand plane formats and the tensor-map helpers shared by
// the tensor-core kernels of libmorl_b200.so (gemm_planes.cu, qhead_envelope.cu); envelope_td.cu uses the mbarrier and bulk-copy
// wrappers.  sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace morl {

// ---- PTX wrappers -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t g_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void g_mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(g_smem_u32(bar)), "r"(count));
}
// once after the last g_mbar_init, before any thread or bulk copy uses the barriers
__device__ __forceinline__ void g_mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void g_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(g_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(g_smem_u32(bar)) : "memory");
}
// Bounded spin: a protocol bug becomes a trap (launch error) instead of a hung GPU.
__device__ __forceinline__ void g_mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    for (uint32_t it = 0; it < (1u << 26); ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(g_smem_u32(bar)), "r"(parity)
            : "memory");
        if (ok) return;
    }
    __trap();
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(g_smem_u32(dst)),
        "l"(map), "r"(g_smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// 1-D bulk copy of `bytes` (a multiple of 16; both addresses 16-byte aligned) from global to shared memory, completing on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(g_smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(g_smem_u32(bar))
                 : "memory");
}
// named barrier `id` over the first `count` threads of the CTA (barrier 0 is __syncthreads)
__device__ __forceinline__ void bar_sync_named(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// ---- TMA / mbarrier ring of the warp-specialised kernels: full[s] (one producer arrival + the transaction bytes) and empty[s] (one
// arrival per consumer warp) for every stage s.  The producer waits on empty[stage] with parity `phase ^ 1`, a consumer on full[stage]
// with `phase`; both walk the stages in the same order.
struct Ring {
    uint32_t depth, stage = 0, phase = 0;
    __device__ __forceinline__ explicit Ring(uint32_t n) : depth(n) {}
    __device__ __forceinline__ void advance() {
        if (++stage == depth) {
            stage = 0;
            phase ^= 1u;
        }
    }
};

// by one thread, before g_mbar_init_fence
__device__ __forceinline__ void init_ring_barriers(uint64_t* full, uint64_t* empty, uint32_t n_stages) {
    for (uint32_t s = 0; s < n_stages; ++s) {
        g_mbar_init(&full[s], 1);
        g_mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
}

// 1 KB alignment (TMA swizzle atoms) by pointer arithmetic ON the shared array, not through an integer cast, so that the compiler keeps
// every derived pointer in the shared address space: through the cast the bias / staging accesses were generic LD.E / ST.E
// (long-scoreboard stalls)
__device__ __forceinline__ uint8_t* align_1k(uint8_t* smem) { return smem + ((1024u - (g_smem_u32(smem) & 1023u)) & 1023u); }

// ---- warpgroup MMA (wgmma.mma_async, sm_90a): D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, both operands through shared-memory descriptors, fp32
// accumulators in the registers of the 128 threads of the warpgroup.  Thread t = 32 w + l of the warpgroup holds, for every 8-column group j,
// d[4 j + {0, 1}] = D[16 w + l / 4][8 j + 2 (l % 4) + {0, 1}] and d[4 j + {2, 3}] = the same columns of row + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// Register re-allocation between the warpgroups of a CTA (setmaxnreg, sm_90a): ptxas budgets a kernel by whole warpgroups, so the
// producer warpgroup gives its registers up and each consumer warpgroup takes a share; every warp of a warpgroup must execute it.
template <int REGS>
__device__ __forceinline__ void warpgroup_reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS>
__device__ __forceinline__ void warpgroup_reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }

#define MORL_WG_R16_0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define MORL_WG_R16_1 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define MORL_WG_R16_2 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define MORL_WG_R16_3 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define MORL_WG_R16_4 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define MORL_WG_R16_5 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define MORL_WG_R16_6 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define MORL_WG_R16_7 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define MORL_WG_A8(d, o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define MORL_WG_A16(d, o) MORL_WG_A8(d, o), MORL_WG_A8(d, o + 8)
#define MORL_WG_REGS_16 "%0, %1, %2, %3, %4, %5, %6, %7"
#define MORL_WG_ACCS_16 MORL_WG_A8(d, 0)
#define MORL_WG_REGS_32 MORL_WG_R16_0
#define MORL_WG_ACCS_32 MORL_WG_A16(d, 0)
#define MORL_WG_REGS_64 MORL_WG_R16_0 ", " MORL_WG_R16_1
#define MORL_WG_ACCS_64 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16)
#define MORL_WG_REGS_96 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2
#define MORL_WG_ACCS_96 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32)
#define MORL_WG_REGS_128 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2 ", " MORL_WG_R16_3
#define MORL_WG_ACCS_128 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32), MORL_WG_A16(d, 48)
#define MORL_WG_REGS_160 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2 ", " MORL_WG_R16_3 ", " MORL_WG_R16_4
#define MORL_WG_ACCS_160 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32), MORL_WG_A16(d, 48), MORL_WG_A16(d, 64)
#define MORL_WG_REGS_192 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2 ", " MORL_WG_R16_3 ", " MORL_WG_R16_4 ", " MORL_WG_R16_5
#define MORL_WG_ACCS_192 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32), MORL_WG_A16(d, 48), MORL_WG_A16(d, 64), MORL_WG_A16(d, 80)
#define MORL_WG_REGS_224 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2 ", " MORL_WG_R16_3 ", " MORL_WG_R16_4 ", " MORL_WG_R16_5 ", " MORL_WG_R16_6
#define MORL_WG_ACCS_224 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32), MORL_WG_A16(d, 48), MORL_WG_A16(d, 64), MORL_WG_A16(d, 80), MORL_WG_A16(d, 96)
#define MORL_WG_REGS_256 MORL_WG_R16_0 ", " MORL_WG_R16_1 ", " MORL_WG_R16_2 ", " MORL_WG_R16_3 ", " MORL_WG_R16_4 ", " MORL_WG_R16_5 ", " MORL_WG_R16_6 ", " MORL_WG_R16_7
#define MORL_WG_ACCS_256 MORL_WG_A16(d, 0), MORL_WG_A16(d, 16), MORL_WG_A16(d, 32), MORL_WG_A16(d, 48), MORL_WG_A16(d, 64), MORL_WG_A16(d, 80), MORL_WG_A16(d, 96), MORL_WG_A16(d, 112)
// TYPE_: "f16" / "bf16"; the N / 2 accumulator registers come first, IA_.. are the operand numbers after them.  `accumulate` = 0 overwrites D.
#define MORL_WGMMA_ASM(N_, TYPE_, IA_, IB_, IP_, ITA_, ITB_)                                                                     \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IP_ ", 0;\n\t"                                                       \
                 "wgmma.mma_async.sync.aligned.m64n" #N_ "k16.f32." TYPE_ "." TYPE_ " {" MORL_WG_REGS_##N_ "}, %" #IA_ ", %" #IB_   \
                 ", p, 1, 1, %" #ITA_ ", %" #ITB_ ";\n\t}"                                                                        \
                 : MORL_WG_ACCS_##N_                                                                                             \
                 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB))
template <int N>
struct Wgmma;
// FMT: plane format (f16x2 -> f16 operands, bf16x3 -> bf16); TA / TB = 1: the operand is MN-major ("transposed") in shared memory
#define MORL_WGMMA_DEF(N_, IA_, IB_, IP_, ITA_, ITB_)                                                          \
    template <>                                                                                                \
    struct Wgmma<N_> {                                                                                         \
        template <int FMT, int TA, int TB>                                                                     \
        __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {  \
            if (FMT == MORL_FMT_F16X2)                                                                         \
                MORL_WGMMA_ASM(N_, "f16", IA_, IB_, IP_, ITA_, ITB_);                                          \
            else                                                                                               \
                MORL_WGMMA_ASM(N_, "bf16", IA_, IB_, IP_, ITA_, ITB_);                                         \
        }                                                                                                      \
    };
MORL_WGMMA_DEF(16, 8, 9, 10, 11, 12)
MORL_WGMMA_DEF(32, 16, 17, 18, 19, 20)
MORL_WGMMA_DEF(64, 32, 33, 34, 35, 36)
MORL_WGMMA_DEF(96, 48, 49, 50, 51, 52)
MORL_WGMMA_DEF(128, 64, 65, 66, 67, 68)
MORL_WGMMA_DEF(160, 80, 81, 82, 83, 84)
MORL_WGMMA_DEF(192, 96, 97, 98, 99, 100)
MORL_WGMMA_DEF(224, 112, 113, 114, 115, 116)
MORL_WGMMA_DEF(256, 128, 129, 130, 131, 132)

// ---- operand formats ------------------------------------------------------------------------------------------------------
template <int FMT>
struct PlaneFmt;

template <>
struct PlaneFmt<MORL_FMT_BF16X3> {
    static constexpr int P = 3, NPROD = 6;
    static constexpr int BK = 32;                                  // 16-bit elements per K-major stage row (64-byte swizzle)
    static constexpr uint32_t kOnes2 = 0x3F803F80u;                // two packed 1.0
    static constexpr int kStages = 2, kStagesMn = 3;
    // small terms first: A2B0, A0B2, A1B1, A1B0, A0B1, A0B0
    __device__ static constexpr int pa(int t) { return t == 0 ? 2 : (t == 2 || t == 3) ? 1 : 0; }
    __device__ static constexpr int pb(int t) { return t == 1 ? 2 : (t == 2 || t == 4) ? 1 : 0; }
    // (a, b) -> P words, word p = plane p of a (low half) and b (high half)
    __device__ __forceinline__ static void split2(float a, float b, uint32_t (&w)[3], float&) {
        const __nv_bfloat16 a0 = __float2bfloat16_rn(a), b0 = __float2bfloat16_rn(b);
        const float ra = a - __bfloat162float(a0), rb = b - __bfloat162float(b0);
        const __nv_bfloat16 a1 = __float2bfloat16_rn(ra), b1 = __float2bfloat16_rn(rb);
        const float sa = ra - __bfloat162float(a1), sb = rb - __bfloat162float(b1);
        const __nv_bfloat16 a2 = __float2bfloat16_rn(sa), b2 = __float2bfloat16_rn(sb);
        w[0] = (uint32_t)__bfloat16_as_ushort(a0) | ((uint32_t)__bfloat16_as_ushort(b0) << 16);
        w[1] = (uint32_t)__bfloat16_as_ushort(a1) | ((uint32_t)__bfloat16_as_ushort(b1) << 16);
        w[2] = (uint32_t)__bfloat16_as_ushort(a2) | ((uint32_t)__bfloat16_as_ushort(b2) << 16);
    }
    __device__ __forceinline__ static void split1(float a, uint16_t (&h)[3], float&) {
        const __nv_bfloat16 a0 = __float2bfloat16_rn(a);
        const float ra = a - __bfloat162float(a0);
        const __nv_bfloat16 a1 = __float2bfloat16_rn(ra);
        const __nv_bfloat16 a2 = __float2bfloat16_rn(ra - __bfloat162float(a1));
        h[0] = __bfloat16_as_ushort(a0); h[1] = __bfloat16_as_ushort(a1); h[2] = __bfloat16_as_ushort(a2);
    }
    __device__ __forceinline__ static void add8(float (&acc)[8], const uint4 v) {  // += eight packed elements of one plane
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            acc[2 * q] += __uint_as_float(w[q] << 16);
            acc[2 * q + 1] += __uint_as_float(w[q] & 0xFFFF0000u);
        }
    }
};

template <>
struct PlaneFmt<MORL_FMT_F16X2> {
    static constexpr int P = 2, NPROD = 3;
    static constexpr int BK = 64;                                  // 128-byte swizzle rows
    static constexpr uint32_t kOnes2 = 0x3C003C00u;
    static constexpr int kStages = 2, kStagesMn = 4;
    // small terms first: A1B0, A0B1, A0B0
    __device__ static constexpr int pa(int t) { return t == 0 ? 1 : 0; }
    __device__ static constexpr int pb(int t) { return t == 1 ? 1 : 0; }
    // `amax` tracks max |a| of the (already scaled) values, for the fp16-range check
    __device__ __forceinline__ static void split2(float a, float b, uint32_t (&w)[2], float& amax) {
        amax = fmaxf(amax, fmaxf(fabsf(a), fabsf(b)));
        const __half2 h0 = __floats2half2_rn(a, b);
        const float2 f0 = __half22float2(h0);
        const __half2 h1 = __floats2half2_rn(a - f0.x, b - f0.y);
        w[0] = *reinterpret_cast<const uint32_t*>(&h0);
        w[1] = *reinterpret_cast<const uint32_t*>(&h1);
    }
    __device__ __forceinline__ static void split1(float a, uint16_t (&h)[2], float& amax) {
        amax = fmaxf(amax, fabsf(a));
        const __half h0 = __float2half_rn(a);
        const __half h1 = __float2half_rn(a - __half2float(h0));
        h[0] = __half_as_ushort(h0); h[1] = __half_as_ushort(h1);
    }
    __device__ __forceinline__ static void add8(float (&acc)[8], const uint4 v) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[q]));
            acc[2 * q] += f.x;
            acc[2 * q + 1] += f.y;
        }
    }
};

__device__ __forceinline__ float ld_scale(const float* p) { return p ? __ldg(p) : 1.0f; }

// Shared-memory matrix descriptor of wgmma, K-major canonical layout with ROWB-byte rows = the swizzle
// span (64 B -> SWIZZLE_64B, 128 B -> SWIZZLE_128B); 8-row groups are contiguous: SBO = 8 * ROWB; LBO unused (1).  A K step of 16
// elements inside the swizzle span is a +32 B advance of the start address.
template <int ROWB>
__device__ __forceinline__ uint64_t make_desc_k(uint32_t smem_addr) {
    static_assert(ROWB == 64 || ROWB == 128, "swizzle span");
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);        // start address, 16-byte units
    d |= (uint64_t)1 << 16;                            // leading byte offset (ignored for swizzled K-major), 16-byte units
    d |= (uint64_t)((8 * ROWB) >> 4) << 32;            // stride byte offset: 8 rows x ROWB
    d |= (uint64_t)(ROWB == 64 ? 2 : 1) << 62;         // swizzle mode: 128 B = 1, 64 B = 2
    return d;
}

// ---- host side: tensor maps through the driver entry point (no link-time dependency on libcuda) ----------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
        else
            (void)cudaGetLastError();
    }
    return fn;
}

static inline int fmt_planes(int fmt) { return fmt == MORL_FMT_F16X2 ? 2 : 3; }
static inline int fmt_bk(int fmt) { return fmt == MORL_FMT_F16X2 ? PlaneFmt<MORL_FMT_F16X2>::BK : PlaneFmt<MORL_FMT_BF16X3>::BK; }
static inline CUtensorMapDataType fmt_tm_type(int fmt) { return fmt == MORL_FMT_F16X2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }

// [P][rows][K] plane tensor, box = P (or one plane) x box_rows x box_k elements, swizzle span = box_k * 2 bytes (64 or 128)
static inline int make_plane_map(CUtensorMap* map, int fmt, const void* base, int rows, int K, long long plane_stride_elems, int box_rows, int box_k,
                                 bool one_plane = false) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return -1;
    const cuuint32_t P = (cuuint32_t)fmt_planes(fmt);
    const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, P};
    const cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)plane_stride_elems * 2};
    const cuuint32_t box[3] = {(cuuint32_t)box_k, (cuuint32_t)box_rows, one_plane ? 1u : P};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(map, fmt_tm_type(fmt), 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           box_k == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

}  // namespace morl
