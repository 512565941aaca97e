// qhead_envelope.cu -- the output layer of BOTH Q-networks, the envelope operator and the vector Bellman target as ONE kernel, sm_90a.
//
// Replaces, for the two no-grad passes of Envelope.update (reference multi_policy/envelope/envelope.py:420 online net on s', :429 target
// net on s', :422-440 einsum -> max -> argmax -> gather x2, :298 Bellman line), the chain
//     Q_on = h_on . W_on^T + b_on   (GEMM, 6.3 MB written)      Q_tg = h_tg . W_tg^T + b_tg   (GEMM, 6.3 MB written)
//     target = envelope_td(Q_on, Q_tg, ...)                     (12.6 MB read)
// by one pass over the last hidden activations: the Q tiles live in registers and shared memory only (SURVEY 8(f)2, hypothesis H1).
//
// One persistent CTA per SM, 288 threads, a tile = 128 pair rows (b*W + j) = 128 / W whole transitions:
//   warp 8   : TMA producer  -- the output-layer weight planes of both nets ONCE per CTA (resident: 2 x K/64 boxes of [2 x 32 x 64]
//              fp16), then per tile and per net K/64 activation boxes [2 planes x 128 rows x 64] through a ring (128-byte swizzle);
//   warps 0-3: group 0       -- the warpgroup issues, for Q_on, 2 (row halves) x 3 x K/16 wgmma.mma_async (M = 64, N = 32, K = 16; products
//   warps 4-7: group 1          A1B0 + A0B1 + A0B0 in the order of gemm_planes_kernel, so the accumulators are bit-identical to the unfused
//              output-layer GEMM), then x 1/(sA sB) + bias, fp32 rows into the shared Q tile (AoS [j][a][d], exactly the layout of Q[b]
//              in HBM); same for Q_tg in group 1.  Then each group runs the envelope scan
//              (envelope_wp.cuh: weight-pair FMA-chain filter + exact re-check, first-occurrence ties) of the transitions t = group,
//              group + 2, ... of the tile and writes  r + (1 - done) gamma Q_tg[b, j*, a*, :].  The producer stages the next tile meanwhile.
// HBM traffic: the activation planes of both nets (2 x 4 B x B W x K), read once; roofline = HBM (DESIGN.md section 4.1b).
#include <stdlib.h>

#include "gemm_tc.cuh"
#include "envelope_wp.cuh"

namespace morl {

constexpr int kQhThreads = 288;   // warps 0-7: two warpgroups (one per network), warp 8: TMA producer
constexpr int kQhBM = 128;
constexpr int kQhBN = 32;       // accumulator columns per net (N = A*D <= 32)
constexpr int kQhMaxStages = 6;

struct QHeadArgs {
    int B, W, A, K, N;            // transitions, weights per transition, actions, hidden width, N = A*D
    int n_tiles;                  // B*W / 128
    int n_stages;                 // depth of the activation ring
    const float* bias[2];         // [N] online / target
    const float* a_scale[2];      // device scalars (powers of two) of the operand planes, nullptr = 1
    const float* b_scale[2];
    const float* wset;            // [W, D]
    const float* reward;          // [B, D]
    const float* done;            // [B]
    float gamma;
    int row_order;
    int reverse;
    int pdl;
    float* target_out;            // [W*B, D]
    int32_t* pref_out;            // [W*B] or nullptr
    int32_t* act_out;             // [W*B] or nullptr
    float* q_out[2];              // optional fp32 copies of the Q tiles [B*W, N] (validation against the unfused path), or nullptr
    int n_nets;                   // 2: the fused operator; 1: output layer of ONE net only, Q written to q_out[0] (morl_qhead_gemm_f32)
};

// shared-memory plan (host and device agree through this)
template <int FMT>
struct QhPlan {
    using F = PlaneFmt<FMT>;
    static constexpr uint32_t kRowB = F::BK * 2;
    static constexpr uint32_t kAStage = F::P * kQhBM * kRowB;    // one activation box
    static constexpr uint32_t kBChunk = F::P * kQhBN * kRowB;    // one weight box (one K block of one net)
    uint32_t off_a, off_q, off_scr, off_bias, off_bar, bytes;
    __host__ __device__ QhPlan(int K, int N, int n_stages) {
        const uint32_t n_kblk = (uint32_t)(K / F::BK);
        off_a = 2u * n_kblk * kBChunk;                             // weights first: [net][kblk]
        off_q = off_a + (uint32_t)n_stages * kAStage;
        off_scr = off_q + ((2u * kQhBM * (uint32_t)N * 4u + 15u) & ~15u);
        off_bias = off_scr + 2u * (((uint32_t)sizeof(wp::Scratch) + 15u) & ~15u);
        off_bar = off_bias + 2u * kQhBN * 4u;
        bytes = off_bar + 256u + 1024u;                           // + alignment slack of the dynamic segment
    }
};

__device__ __forceinline__ void bar_sync_named(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

template <int FMT, int D, int MODE>
__global__ void __launch_bounds__(kQhThreads, 1)
qhead_envelope_kernel(const __grid_constant__ CUtensorMap tmA_on, const __grid_constant__ CUtensorMap tmA_tg, const __grid_constant__ CUtensorMap tmB_on,
                      const __grid_constant__ CUtensorMap tmB_tg, const QHeadArgs g) {
    using F = PlaneFmt<FMT>;
    using L = QhPlan<FMT>;
    constexpr int BK = F::BK;
    constexpr uint32_t ROWB = L::kRowB;
    const L plan(g.K, g.N, g.n_stages);
    const uint32_t kStages = (uint32_t)g.n_stages;
    const int n_kblk = g.K / BK;
    extern __shared__ uint8_t qsmem_raw[];
    uint8_t* sm = qsmem_raw + ((1024u - (g_smem_u32(qsmem_raw) & 1023u)) & 1023u);  // (pointer arithmetic on the shared array: see gemm_planes.cu)
    uint8_t* smB = sm;
    uint8_t* smA = sm + plan.off_a;
    float* Qst = reinterpret_cast<float*>(sm + plan.off_q);  // [2 nets][128 rows][N]
    wp::Scratch* scr = reinterpret_cast<wp::Scratch*>(sm + plan.off_scr);
    float* bias_s = reinterpret_cast<float*>(sm + plan.off_bias);  // [2][32]
    uint64_t* full = reinterpret_cast<uint64_t*>(sm + plan.off_bar);
    uint64_t* empty = full + kQhMaxStages;
    uint64_t* bfull = empty + kQhMaxStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int N = g.N;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) {
            g_mbar_init(&full[s], 1);
            g_mbar_init(&empty[s], 8);  // one arrival per consumer warp (both groups walk every stage)
        }
        g_mbar_init(bfull, 1);
        g_mbar_init_fence();
    }
    if (g.pdl) {  // nothing above reads global memory; everything below may (see gemm_planes_kernel)
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    if (threadIdx.x < 2 * kQhBN) {
        const int net = threadIdx.x >> 5, n = threadIdx.x & 31;
        bias_s[threadIdx.x] = (g.bias[net] && n < N) ? g.bias[net][n] : 0.f;
    }
    __syncthreads();

    if (warp == 8) {
        // ================= TMA producer =================
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_on) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_tg) : "memory");
            g_mbar_expect_tx(bfull, (uint32_t)g.n_nets * (uint32_t)n_kblk * L::kBChunk);
            for (int net = 0; net < g.n_nets; ++net)
                for (int kb = 0; kb < n_kblk; ++kb)
                    tma_load_3d(smB + (uint32_t)(net * n_kblk + kb) * L::kBChunk, net ? &tmB_tg : &tmB_on, bfull, kb * BK, 0, 0);
            uint32_t stage = 0, phase = 0;
            for (int u = blockIdx.x; u < g.n_tiles; u += gridDim.x) {
                const int tile = g.reverse ? g.n_tiles - 1 - u : u;
                for (int net = 0; net < g.n_nets; ++net) {
                    for (int kb = 0; kb < n_kblk; ++kb) {
                        g_mbar_wait(&empty[stage], phase ^ 1u);
                        g_mbar_expect_tx(&full[stage], L::kAStage);
                        tma_load_3d(smA + stage * L::kAStage, net ? &tmA_tg : &tmA_on, &full[stage], kb * BK, tile * kQhBM, 0);
                        if (++stage == kStages) {
                            stage = 0;
                            phase ^= 1u;
                        }
                    }
                }
            }
        }
    } else {
        // ================= MMA + epilogue + envelope scan (warpgroups 0 and 1) =================
        const int grp = warp >> 2;                   // 0: computes and stages Q_on, 1: Q_tg; scans the transitions t = grp, grp + 2, ...
        const int tid_g = (warp & 3) * 32 + lane;    // index in the group (scan / finish roles)
        const int l4 = lane & 3;
        const float k_acc = 1.0f / (ld_scale(g.a_scale[grp]) * ld_scale(g.b_scale[grp]));
        const int W = g.W, A = g.A, C = W * A, T = kQhBM / W;
        const bool fused = g.n_nets == 2;
        wp::Role<D> role;
        if (fused) wp::load_role<D>(role, g.wset, W, tid_g);
        const int part = tid_g & 1;
        auto sync_g = [&]() { bar_sync_named(2 + grp, 128); };
        constexpr uint32_t a_plane = kQhBM * ROWB, b_plane = kQhBN * ROWB;
        if (grp < g.n_nets) g_mbar_wait(bfull, 0);
        uint32_t stage = 0, phase = 0;
        for (int u = blockIdx.x; u < g.n_tiles; u += gridDim.x) {
            const int tile = g.reverse ? g.n_tiles - 1 - u : u;
            // acc[mh]: rows [64 mh, 64 mh + 64) of the tile, 32 columns: the products of a K step in the order of gemm_planes_kernel, so the
            // accumulators are bit-identical to the unfused output-layer GEMM.  Both groups walk EVERY stage of the ring in order (a parity
            // wait is only meaningful one phase ahead) and release it; a group issues MMAs on the stages of its own net only.
            float acc[2][16];
            for (int net = 0; net < g.n_nets; ++net) {
                uint32_t prev = 0;
                for (int kb = 0; kb < n_kblk; ++kb) {
                    g_mbar_wait(&full[stage], phase);
                    if (net == grp) {
                        wgmma_fence();
                        const uint32_t a0 = g_smem_u32(smA + stage * L::kAStage);
                        const uint32_t b0 = g_smem_u32(smB + (uint32_t)(grp * n_kblk + kb) * L::kBChunk);
#pragma unroll
                        for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
                            for (int ks = 0; ks < BK / 16; ++ks) {
#pragma unroll
                                for (int t = 0; t < F::NPROD; ++t) {
                                    const uint64_t ad = make_desc_k<ROWB>(a0 + F::pa(t) * a_plane + (uint32_t)mh * 64u * ROWB + ks * 32);
                                    const uint64_t bd = make_desc_k<ROWB>(b0 + F::pb(t) * b_plane + ks * 32);
                                    Wgmma<kQhBN>::template mma<FMT, 0, 0>(acc[mh], ad, bd, (kb | ks | t) != 0 ? 1u : 0u);
                                }
                            }
                        }
                        wgmma_commit();
                        if (kb > 0) {
                            wgmma_wait<1>();
                            if (lane == 0) g_mbar_arrive(&empty[prev]);  // frees the activation stage when the MMAs above have read it
                        }
                        prev = stage;
                    } else if (lane == 0) {
                        g_mbar_arrive(&empty[stage]);  // the other group's operand
                    }
                    if (++stage == kStages) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
                if (net == grp) {
                    wgmma_wait<0>();
                    if (lane == 0) g_mbar_arrive(&empty[prev]);
                }
            }
            if (!fused) {
                // output layer of one net: the rows go straight to HBM
                if (grp == 0) {
#pragma unroll
                    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int row = mh * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
                            float* orow = g.q_out[0] + ((size_t)tile * kQhBM + row) * N;
#pragma unroll
                            for (int q = 0; q < 4; ++q)
#pragma unroll
                                for (int c = 0; c < 2; ++c) {
                                    const int col = 8 * q + 2 * l4 + c;
                                    if (col < N) orow[col] = __fmaf_rn(acc[mh][4 * q + 2 * h + c], k_acc, bias_s[col]);
                                }
                        }
                }
                continue;
            }
            bar_sync_named(1, 256);  // every scan of the previous tile has finished reading the Q tile
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = mh * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
                    float* qrow = Qst + ((size_t)grp * kQhBM + row) * N;
                    float* orow = g.q_out[grp] ? g.q_out[grp] + ((size_t)tile * kQhBM + row) * N : nullptr;
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            const int col = 8 * q + 2 * l4 + c;
                            if (col < N) {
                                const float x = __fmaf_rn(acc[mh][4 * q + 2 * h + c], k_acc, bias_s[grp * kQhBN + col]);
                                qrow[col] = x;
                                if (orow) orow[col] = x;
                            }
                        }
                }
            bar_sync_named(1, 256);  // both Q tiles are staged
            for (int t = grp; t < T; t += 2) {
                const int b = tile * T + t;
                const float* Qa = Qst + (size_t)t * W * N;
                const float* Qt = Qst + ((size_t)kQhBM + (size_t)t * W) * N;
                float rw[D];
                const float dn = __ldg(g.done + b);
#pragma unroll
                for (int r = 0; r < D; ++r) rw[r] = __ldg(g.reward + (size_t)b * D + r);
                const int cstar = wp::scan_transition<D, MODE>(Qa, scr[grp], role, tid_g, C, sync_g);
                if (role.f_active) {
                    const size_t k = (g.row_order == MORL_ROWS_REFERENCE) ? ((size_t)role.fi * g.B + b) : ((size_t)b * W + role.fi);
                    if (part == 0) {
                        const float* qt = Qt + (size_t)cstar * D;
#pragma unroll
                        for (int r = 0; r < D; ++r) g.target_out[k * D + r] = bellman(rw[r], dn, g.gamma, qt[r]);
                    } else {
                        const int jstar = cstar / A;
                        if (g.pref_out) g.pref_out[k] = jstar;
                        if (g.act_out) g.act_out[k] = cstar - jstar * A;
                    }
                }
                if (t + 2 < T) sync_g();  // the group's scratch is rewritten by its next transition
            }
        }
    }
}

template <int FMT, int D, int MODE>
static int launch_qhead(const CUtensorMap& tmA_on, const CUtensorMap& tmA_tg, const CUtensorMap& tmB_on, const CUtensorMap& tmB_tg, const QHeadArgs& g,
                        size_t smem, int grid, cudaStream_t st) {
    static bool attr_set = false;
    auto kern = qhead_envelope_kernel<FMT, D, MODE>;
    if (!attr_set) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        attr_set = true;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kQhThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g.pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kern, tmA_on, tmA_tg, tmB_on, tmB_tg, g);
    return check_launch("morl_qhead_envelope_td_f32");
}

}  // namespace morl

extern "C" int morl_qhead_envelope_supported(int fmt, int B, int W, int A, int D, int K) {
    using namespace morl;
    if (fmt != MORL_FMT_F16X2) return 0;
    if (B <= 0 || W <= 0 || A <= 0 || D < 2 || D > 4 || K <= 0) return 0;
    if (W > 64 || (kQhBM % W) != 0 || ((long long)B * W) % kQhBM != 0) return 0;
    if (A * D > kQhBN || (W * A) % 16 != 0 || (W * A * D) % 4 != 0) return 0;
    if (K % PlaneFmt<MORL_FMT_F16X2>::BK != 0 || K > 256) return 0;
    return 1;
}

extern "C" int morl_qhead_envelope_td_f32(int fmt, const void* a_on_planes, const void* a_tg_planes, long long a_plane_stride, const float* a_scale_on,
                                          const float* a_scale_tg, const void* w_on_planes, const void* w_tg_planes, long long w_plane_stride,
                                          const float* w_scale_on, const float* w_scale_tg, const float* bias_on, const float* bias_tg, int K,
                                          const float* wset, const float* reward, const float* done, float gamma, int B, int W, int A, int D,
                                          int dot_mode, int row_order, int reverse_tiles, float* target_out, int32_t* pref_out, int32_t* act_out,
                                          float* q_on_out, float* q_tg_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(a_on_planes && a_tg_planes && w_on_planes && w_tg_planes && wset && reward && done && target_out, MORL_ERR_NULL,
                 "morl_qhead_envelope_td_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && A > 0 && D > 0 && K > 0, MORL_ERR_SHAPE, "morl_qhead_envelope_td_f32: bad shape B=%d W=%d A=%d D=%d K=%d", B, W, A, D, K);
    MORL_REQUIRE(morl_qhead_envelope_supported(fmt, B, W, A, D, K), MORL_ERR_UNSUPPORTED,
                 "morl_qhead_envelope_td_f32: unsupported configuration fmt=%d B=%d W=%d A=%d D=%d K=%d (need f16x2 planes, W <= 64 dividing 128, "
                 "B*W %% 128 == 0, A*D <= 32, W*A %% 16 == 0, W*A*D %% 4 == 0, 2 <= D <= 4, K %% 64 == 0, K <= 256)",
                 fmt, B, W, A, D, K);
    MORL_REQUIRE(dot_mode >= 0 && dot_mode <= 2, MORL_ERR_UNSUPPORTED, "morl_qhead_envelope_td_f32: bad dot_mode %d", dot_mode);
    MORL_REQUIRE(row_order == MORL_ROWS_REFERENCE || row_order == MORL_ROWS_BMAJOR, MORL_ERR_UNSUPPORTED, "morl_qhead_envelope_td_f32: bad row_order %d",
                 row_order);
    MORL_REQUIRE(aligned16(a_on_planes) && aligned16(a_tg_planes) && aligned16(w_on_planes) && aligned16(w_tg_planes), MORL_ERR_ALIGN,
                 "morl_qhead_envelope_td_f32: operand planes must be 16-byte aligned");
    constexpr int kFmt = MORL_FMT_F16X2;
    constexpr int BK = PlaneFmt<kFmt>::BK;
    const int M = B * W;
    CUtensorMap tmA_on, tmA_tg, tmB_on, tmB_tg;
    int rc = make_plane_map(&tmA_on, fmt, a_on_planes, M, K, a_plane_stride, kQhBM, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_envelope_td_f32: cuTensorMapEncodeTiled(A online) failed (%d)", rc);
    rc = make_plane_map(&tmA_tg, fmt, a_tg_planes, M, K, a_plane_stride, kQhBM, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_envelope_td_f32: cuTensorMapEncodeTiled(A target) failed (%d)", rc);
    rc = make_plane_map(&tmB_on, fmt, w_on_planes, kQhBN, K, w_plane_stride, kQhBN, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_envelope_td_f32: cuTensorMapEncodeTiled(W online) failed (%d)", rc);
    rc = make_plane_map(&tmB_tg, fmt, w_tg_planes, kQhBN, K, w_plane_stride, kQhBN, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_envelope_td_f32: cuTensorMapEncodeTiled(W target) failed (%d)", rc);
    QHeadArgs g;
    memset(&g, 0, sizeof(g));
    g.B = B; g.W = W; g.A = A; g.K = K; g.N = A * D;
    g.n_tiles = M / kQhBM;
    g.bias[0] = bias_on; g.bias[1] = bias_tg;
    g.a_scale[0] = a_scale_on; g.a_scale[1] = a_scale_tg;
    g.b_scale[0] = w_scale_on; g.b_scale[1] = w_scale_tg;
    g.wset = wset; g.reward = reward; g.done = done; g.gamma = gamma;
    g.row_order = row_order; g.reverse = reverse_tiles ? 1 : 0;
    g.target_out = target_out; g.pref_out = pref_out; g.act_out = act_out;
    g.q_out[0] = q_on_out; g.q_out[1] = q_tg_out;
    g.n_nets = 2;
    static const bool want_pdl = [] { const char* e = getenv("MORL_GEMM_PDL"); return !(e && e[0] == '0'); }();
    g.pdl = want_pdl ? 1 : 0;
    // activation ring: as many stages as fit beside the resident weight planes, the Q tiles and the scan scratch
    int n_st = kQhMaxStages;
    static const int st_env = [] { const char* e = getenv("MORL_QHEAD_STAGES"); return e ? atoi(e) : 0; }();
    if (st_env > 0 && st_env < n_st) n_st = st_env;
    while (n_st > 1 && QhPlan<kFmt>(K, g.N, n_st).bytes > 227u * 1024u) --n_st;
    MORL_REQUIRE(QhPlan<kFmt>(K, g.N, n_st).bytes <= 227u * 1024u, MORL_ERR_UNSUPPORTED, "morl_qhead_envelope_td_f32: shared-memory plan does not fit");
    g.n_stages = n_st;
    const size_t smem = QhPlan<kFmt>(K, g.N, n_st).bytes;
    int sms = morl_device_sm_count();
    if (sms <= 0) sms = 132;
    const int grid = g.n_tiles < sms ? g.n_tiles : sms;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    bool launched = false;
    int ret = MORL_OK;
    switch (D) {
        case 2: { constexpr int kD = 2; MORL_DISPATCH_MODE(dot_mode, { ret = launch_qhead<kFmt, kD, kMode>(tmA_on, tmA_tg, tmB_on, tmB_tg, g, smem, grid, st); launched = true; }); } break;
        case 3: { constexpr int kD = 3; MORL_DISPATCH_MODE(dot_mode, { ret = launch_qhead<kFmt, kD, kMode>(tmA_on, tmA_tg, tmB_on, tmB_tg, g, smem, grid, st); launched = true; }); } break;
        case 4: { constexpr int kD = 4; MORL_DISPATCH_MODE(dot_mode, { ret = launch_qhead<kFmt, kD, kMode>(tmA_on, tmA_tg, tmB_on, tmB_tg, g, smem, grid, st); launched = true; }); } break;
        default: break;
    }
    MORL_REQUIRE(launched, MORL_ERR_UNSUPPORTED, "morl_qhead_envelope_td_f32: no kernel for D=%d mode=%d", D, dot_mode);
    return ret;
}

extern "C" int morl_qhead_gemm_supported(int fmt, int M, int N, int K) {
    using namespace morl;
    return fmt == MORL_FMT_F16X2 && M > 0 && M % kQhBM == 0 && N > 0 && N <= kQhBN && K > 0 && K % PlaneFmt<MORL_FMT_F16X2>::BK == 0 && K <= 256;
}

// Output layer of ONE network, Q = A . W^T + b written as fp32 rows: the narrow-N form of morl_gemm_planes_f32 (same accumulation order: bit-identical)
// with the weight planes resident in shared memory and a deep activation ring -- the kernel above without its operator half.
extern "C" int morl_qhead_gemm_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* w_planes,
                                   long long w_plane_stride, const float* w_scale, const float* bias, int M, int N, int K, int reverse_tiles, float* q_out,
                                   void* stream) {
    using namespace morl;
    MORL_REQUIRE(a_planes && w_planes && q_out, MORL_ERR_NULL, "morl_qhead_gemm_f32: NULL pointer argument");
    MORL_REQUIRE(morl_qhead_gemm_supported(fmt, M, N, K), MORL_ERR_UNSUPPORTED,
                 "morl_qhead_gemm_f32: unsupported configuration fmt=%d M=%d N=%d K=%d (need f16x2 planes, M %% 128 == 0, N <= 32, K %% 64 == 0, K <= 256)", fmt, M,
                 N, K);
    MORL_REQUIRE(aligned16(a_planes) && aligned16(w_planes) && aligned16(q_out), MORL_ERR_ALIGN, "morl_qhead_gemm_f32: operands must be 16-byte aligned");
    constexpr int kFmt = MORL_FMT_F16X2;
    constexpr int BK = PlaneFmt<kFmt>::BK;
    CUtensorMap tmA, tmB;
    int rc = make_plane_map(&tmA, fmt, a_planes, M, K, a_plane_stride, kQhBM, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_gemm_f32: cuTensorMapEncodeTiled(A) failed (%d)", rc);
    rc = make_plane_map(&tmB, fmt, w_planes, kQhBN, K, w_plane_stride, kQhBN, BK);
    MORL_REQUIRE(rc == 0, MORL_ERR_NO_DEVICE, "morl_qhead_gemm_f32: cuTensorMapEncodeTiled(W) failed (%d)", rc);
    QHeadArgs g;
    memset(&g, 0, sizeof(g));
    g.B = M / kQhBM; g.W = kQhBM; g.A = 1; g.K = K; g.N = N;  // (B, W, A are not used without the operator half)
    g.n_tiles = M / kQhBM;
    g.bias[0] = bias;
    g.a_scale[0] = a_scale; g.b_scale[0] = w_scale;
    g.reverse = reverse_tiles ? 1 : 0;
    g.q_out[0] = q_out;
    g.n_nets = 1;
    static const bool want_pdl = [] { const char* e = getenv("MORL_GEMM_PDL"); return !(e && e[0] == '0'); }();
    g.pdl = want_pdl ? 1 : 0;
    int n_st = kQhMaxStages;
    while (n_st > 1 && QhPlan<kFmt>(K, N, n_st).bytes > 227u * 1024u) --n_st;
    g.n_stages = n_st;
    const size_t smem = QhPlan<kFmt>(K, N, n_st).bytes;
    int sms = morl_device_sm_count();
    if (sms <= 0) sms = 132;
    const int grid = g.n_tiles < sms ? g.n_tiles : sms;
    return launch_qhead<kFmt, 3, MORL_DOT_UNFUSED>(tmA, tmA, tmB, tmB, g, smem, grid, static_cast<cudaStream_t>(stream));
}
