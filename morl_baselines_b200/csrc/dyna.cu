// dyna.cu -- GPI-PD's Dyna planning step on the device (SURVEY 8(f)3).
//
// morl_ensemble_sample_f32 fuses everything between the last EnsembleLayer of the probabilistic ensemble and the imagined transition
// (reference common/model_based/probabilistic_ensemble.py:115-154 + common/model_based/utils.py:162-170):
//     mean, logvar = chunk(out, 2)                                                              (:115)
//     logvar = max_logvar - softplus(max_logvar - logvar);  logvar = min_logvar + softplus(logvar - min_logvar)   (:118-119)
//     samples = mean + exp(0.5 logvar) * noise                                                  (:127-128; noise = th.randn, or none: deterministic)
//     vars = exp(logvar); mean_ens = mean_e(mean); var_ens = mean_e(mean^2 + vars) - mean_ens^2  (:140-147)
//     uncertainty = sum_o sqrt(var_ens + 1e-12)                                                  (:148-149)
//     sample / var of the elite model drawn for the row (model_inds, :143, :152-154), sample[:, rew_dim:] += obs (utils.py:165)
// The reference moves three [E, N, O] tensors to the host and does this in numpy; here the raw [E, N, 2 O] output is read once.
// One warp per row; bound: HBM (E * 2 O * 4 bytes per row read, 2 O * 4 + 4 written).
#include "common.cuh"

namespace morl {

__device__ __forceinline__ float softplus_t(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // torch F.softplus (beta 1, threshold 20)

// Per-row arithmetic of the ensemble sample, shared by morl_ensemble_sample_f32 and morl_dyna_commit_f32 so that both produce the same
// bits.  One warp per row, lanes stride over the O outputs; sink(o, sample, var) receives every column of the drawn model, and the
// return value is the row's uncertainty (butterfly-reduced: every lane holds it).
template <class Sink>
__device__ __forceinline__ float ensemble_row(const float* __restrict__ out, const float* __restrict__ max_logvar, const float* __restrict__ min_logvar,
                                              int pick, const float* __restrict__ noise, const float* __restrict__ obs, int rew_dim, int E, int N, int O,
                                              int n, int lane, Sink&& sink) {
    float unc = 0.f;
    for (int o = lane; o < O; o += 32) {
        const float hi = __ldg(max_logvar + o), lo = __ldg(min_logvar + o);
        float sum_m = 0.f, sum_s = 0.f, s_pick = 0.f, v_pick = 0.f;
        for (int e = 0; e < E; ++e) {
            const float* row = out + ((size_t)e * N + n) * (2 * O);
            const float m = __ldg(row + o);
            float lv = __ldg(row + O + o);
            lv = __fsub_rn(hi, softplus_t(__fsub_rn(hi, lv)));
            lv = __fadd_rn(lo, softplus_t(__fsub_rn(lv, lo)));
            const float var = expf(lv);
            // ensemble moments in the reference's order: sequential sums over the models, one divide at the end (numpy mean over axis 0)
            sum_m = e == 0 ? m : __fadd_rn(sum_m, m);
            const float t = __fadd_rn(__fmul_rn(m, m), var);
            sum_s = e == 0 ? t : __fadd_rn(sum_s, t);
            if (e == pick) {
                v_pick = var;
                s_pick = noise ? __fadd_rn(m, __fmul_rn(expf(__fmul_rn(0.5f, lv)), __ldg(noise + ((size_t)e * N + n) * O + o))) : m;
            }
        }
        const float mean_e = __fdiv_rn(sum_m, (float)E);
        const float var_e = __fsub_rn(__fdiv_rn(sum_s, (float)E), __fmul_rn(mean_e, mean_e));
        unc += sqrtf(__fadd_rn(var_e, 1e-12f));
        if (obs && o >= rew_dim) s_pick = __fadd_rn(s_pick, __ldg(obs + (size_t)n * (O - rew_dim) + (o - rew_dim)));
        sink(o, s_pick, v_pick);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) unc += __shfl_xor_sync(0xffffffffu, unc, off);
    return unc;
}

__global__ void __launch_bounds__(256) ensemble_sample_kernel(const float* __restrict__ out, const float* __restrict__ max_logvar,
                                                              const float* __restrict__ min_logvar, const int32_t* __restrict__ model_idx,
                                                              const float* __restrict__ noise, const float* __restrict__ obs, int rew_dim, int E, int N,
                                                              int O, float* __restrict__ sample_out, float* __restrict__ var_out,
                                                              float* __restrict__ unc_out) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= N) return;
    const int n = warp;
    const float unc = ensemble_row(out, max_logvar, min_logvar, model_idx[n], noise, obs, rew_dim, E, N, O, n, lane, [&](int o, float s, float v) {
        sample_out[(size_t)n * O + o] = s;
        var_out[(size_t)n * O + o] = v;
    });
    if (lane == 0) unc_out[n] = unc;
}

// ---- morl_dyna_commit_f32: one imagined step from the raw ensemble output to rows of the model replay buffer ----------------------------
// Pass 1 (dyna_flags_kernel): per row the sample, the termination rule on (r, s') and the uncertainty gate; per row a flag byte
//   (bit 0 kept, bit 1 alive), per tile of kCommitTile rows the two counts.
// Pass 2 (dyna_write_kernel): every block sums the tile counts (its exclusive prefix and the totals), ranks its rows with warp ballots,
//   recomputes the sample of the rows it has to write (the same ensemble_row call, so the same bits) and scatters them: kept row k goes to
//   ring slot (ptr + k) % capacity when k >= kept - capacity (sequential adds would overwrite the earlier ones), alive row j to next_alive[j].
// Recomputing instead of staging the sample keeps the workspace independent of O; the second read of `out` is L2-resident at the rollout's
// sizes.  Integer counts only: the result does not depend on block scheduling.
constexpr int kCommitTile = 64;   // rows per block in both passes: the scan granularity
constexpr int kCommitWarps = 8;

__device__ __forceinline__ bool term_done(int rule, const float* st, bool bad) {
    // st: s'[0], s'[1], s'[6], s'[7], r[0]; comparisons in float32 as the tensor rules (common/model_based/utils.py), IEEE NaN semantics
    switch (rule) {
        case MORL_TERM_HOPPER: return !(!bad && st[0] > 0.7f && fabsf(st[1]) < 0.2f);
        case MORL_TERM_HUMANOID: return !(1.0f < st[0] && st[0] < 2.0f);
        case MORL_TERM_MOUNTAINCAR: return st[0] >= 0.45f && st[1] >= 0.0f;
        case MORL_TERM_LUNARLANDER: return fabsf(st[0]) >= 1.0f || (st[4] != 0.0f && st[2] >= 0.95f && st[3] >= 0.95f);
        default: return false;
    }
}

__global__ void __launch_bounds__(kCommitWarps * 32) dyna_flags_kernel(const float* __restrict__ out, const float* __restrict__ max_logvar,
                                                                        const float* __restrict__ min_logvar, const int32_t* __restrict__ model_idx,
                                                                        const float* __restrict__ noise, const float* __restrict__ obs, int rew_dim, int E,
                                                                        int N, int O, int rule, float max_uncertainty, float* __restrict__ unc_out,
                                                                        uint8_t* __restrict__ flags, int* __restrict__ tile_counts) {
    __shared__ float stash[kCommitWarps][5];
    __shared__ uint8_t s_flag[kCommitTile];
    __shared__ int s_cnt[2][kCommitTile / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* st = stash[warp];
    for (int r = warp; r < kCommitTile; r += kCommitWarps) {
        const int n = blockIdx.x * kCommitTile + r;
        if (n >= N) {
            if (lane == 0) s_flag[r] = 0;
            continue;
        }
        int bad = 0;  // HOPPER: a non-finite state column, or s'[1:] not < 100
        const float unc = ensemble_row(out, max_logvar, min_logvar, model_idx[n], noise, obs, rew_dim, E, N, O, n, lane, [&](int o, float s, float) {
            const int c = o - rew_dim;
            if (c < 0) {
                if (o == 0) st[4] = s;
                return;
            }
            if (c < 2) st[c] = s;
            else if (c == 6 || c == 7) st[c - 4] = s;
            bad |= (int)(!isfinite(s) || (c >= 1 && !(s < 100.0f)));
        });
        const bool any_bad = __any_sync(0xffffffffu, bad);
        __syncwarp();
        if (lane == 0) {
            const bool keep = unc < max_uncertainty;  // strict, so NaN is never kept
            const bool live = !term_done(rule, st, any_bad);
            const uint8_t f = (uint8_t)(keep | (live << 1));
            flags[n] = f;
            s_flag[r] = f;
            unc_out[n] = unc;
        }
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x < kCommitTile) {
        const uint8_t f = s_flag[threadIdx.x];
        const unsigned kb = __ballot_sync(0xffffffffu, f & 1), ab = __ballot_sync(0xffffffffu, f & 2);
        if (lane == 0) {
            s_cnt[0][warp] = __popc(kb);
            s_cnt[1][warp] = __popc(ab);
        }
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        int t = 0;
        for (int w = 0; w < kCommitTile / 32; ++w) t += s_cnt[threadIdx.x][w];
        tile_counts[2 * blockIdx.x + threadIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kCommitWarps * 32) dyna_write_kernel(
    const float* __restrict__ out, const float* __restrict__ max_logvar, const float* __restrict__ min_logvar, const int32_t* __restrict__ model_idx,
    const float* __restrict__ noise, const float* __restrict__ obs, const float* __restrict__ act, int rew_dim, int E, int N, int O, int A,
    const uint8_t* __restrict__ flags, const int* __restrict__ tile_counts, int n_tiles, float* __restrict__ st_obs, float* __restrict__ st_next_obs,
    float* __restrict__ st_act, float* __restrict__ st_rew, float* __restrict__ st_done, int capacity, int ptr, float* __restrict__ next_alive,
    int32_t* __restrict__ counts_out) {
    __shared__ int s_red[4][kCommitWarps];
    __shared__ int s_warp_tot[2][kCommitTile / 32];
    __shared__ int s_slot[kCommitTile], s_arow[kCommitTile];
    __shared__ uint8_t s_flag[kCommitTile];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, S = O - rew_dim;
    // exclusive prefix of this tile and the totals (every block sums the same integers: no inter-block communication)
    int v[4] = {0, 0, 0, 0};
    for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
        const int k = tile_counts[2 * t], a = tile_counts[2 * t + 1];
        v[2] += k;
        v[3] += a;
        if (t < (int)blockIdx.x) {
            v[0] += k;
            v[1] += a;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], off);
        if (lane == 0) s_red[i][warp] = v[i];
    }
    // in-tile ranks by ballot
    const int r = threadIdx.x;
    bool keep = false, live = false;
    if (r < kCommitTile) {
        const int n = blockIdx.x * kCommitTile + r;
        const uint8_t f = n < N ? flags[n] : (uint8_t)0;
        s_flag[r] = f;
        keep = f & 1;
        live = (f >> 1) & 1;
        const unsigned kb = __ballot_sync(0xffffffffu, keep), ab = __ballot_sync(0xffffffffu, live);
        if (lane == 0) {
            s_warp_tot[0][warp] = __popc(kb);
            s_warp_tot[1][warp] = __popc(ab);
        }
        const unsigned lt = (1u << lane) - 1u;
        v[0] = __popc(kb & lt);
        v[1] = __popc(ab & lt);
    }
    __syncthreads();
    if (r < kCommitTile) {
        int base[4] = {0, 0, 0, 0};
        for (int w = 0; w < kCommitWarps; ++w)
#pragma unroll
            for (int i = 0; i < 4; ++i) base[i] += s_red[i][w];
        for (int w = 0; w < warp; ++w) {
            base[0] += s_warp_tot[0][w];
            base[1] += s_warp_tot[1][w];
        }
        const long long k = (long long)base[0] + v[0];
        s_slot[r] = keep && k >= (long long)base[2] - capacity ? (int)(((long long)ptr + k) % capacity) : -1;
        s_arow[r] = live ? base[1] + v[1] : -1;
        if (blockIdx.x == 0 && r == 0) {
            counts_out[0] = base[2];
            counts_out[1] = base[3];
        }
    }
    __syncthreads();
    for (int rr = warp; rr < kCommitTile; rr += kCommitWarps) {
        const int n = blockIdx.x * kCommitTile + rr;
        if (n >= N) break;
        const int slot = s_slot[rr], arow = s_arow[rr];
        if (slot < 0 && arow < 0) continue;  // warp-uniform
        ensemble_row(out, max_logvar, min_logvar, model_idx[n], noise, obs, rew_dim, E, N, O, n, lane, [&](int o, float s, float) {
            const int c = o - rew_dim;
            if (c < 0) {
                if (slot >= 0) st_rew[(size_t)slot * rew_dim + o] = s;
                return;
            }
            if (slot >= 0) st_next_obs[(size_t)slot * S + c] = s;
            if (arow >= 0) next_alive[(size_t)arow * S + c] = s;
        });
        if (slot >= 0) {
            for (int c = lane; c < S; c += 32) st_obs[(size_t)slot * S + c] = __ldg(obs + (size_t)n * S + c);
            for (int c = lane; c < A; c += 32) st_act[(size_t)slot * A + c] = __ldg(act + (size_t)n * A + c);
            if (lane == 0) st_done[slot] = (s_flag[rr] & 2) ? 0.0f : 1.0f;
        }
    }
}

}  // namespace morl

extern "C" int morl_ensemble_sample_f32(const float* out, const float* max_logvar, const float* min_logvar, const int32_t* model_idx, const float* noise,
                                        const float* obs, int rew_dim, int E, int N, int O, float* sample_out, float* var_out, float* uncertainty_out,
                                        void* stream) {
    using namespace morl;
    MORL_REQUIRE(out && max_logvar && min_logvar && model_idx && sample_out && var_out && uncertainty_out, MORL_ERR_NULL,
                 "morl_ensemble_sample_f32: NULL pointer argument");
    MORL_REQUIRE(E > 0 && N > 0 && O > 0 && rew_dim >= 0 && rew_dim <= O, MORL_ERR_SHAPE, "morl_ensemble_sample_f32: bad shape E=%d N=%d O=%d rew_dim=%d", E, N, O,
                 rew_dim);
    const int warps_per_block = 8;
    const unsigned grid = (unsigned)((N + warps_per_block - 1) / warps_per_block);
    ensemble_sample_kernel<<<grid, warps_per_block * 32, 0, static_cast<cudaStream_t>(stream)>>>(out, max_logvar, min_logvar, model_idx, noise, obs, rew_dim, E, N, O,
                                                                                                 sample_out, var_out, uncertainty_out);
    return check_launch("morl_ensemble_sample_f32");
}

static inline int dyna_commit_tiles(int N) { return (N + morl::kCommitTile - 1) / morl::kCommitTile; }

extern "C" size_t morl_dyna_commit_workspace_bytes(int N) {
    if (N <= 0) return 0;
    const size_t tiles = (size_t)dyna_commit_tiles(N);
    return tiles * 2 * sizeof(int) + (((size_t)N + 15) & ~(size_t)15);
}

extern "C" int morl_dyna_commit_f32(const float* out, const float* max_logvar, const float* min_logvar, const int32_t* model_idx, const float* noise,
                                    const float* obs, const float* act, int rew_dim, int E, int N, int O, int A, int rule, float max_uncertainty,
                                    float* st_obs, float* st_next_obs, float* st_act, float* st_rew, float* st_done, int capacity, int ptr,
                                    float* next_alive, float* uncertainty_out, int32_t* counts_out, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(out && max_logvar && min_logvar && model_idx && obs && act && st_obs && st_next_obs && st_act && st_done && next_alive && uncertainty_out &&
                     counts_out && workspace && (st_rew || rew_dim == 0),
                 MORL_ERR_NULL, "morl_dyna_commit_f32: NULL pointer argument");
    MORL_REQUIRE(E > 0 && N > 0 && A > 0 && rew_dim >= 0 && O > rew_dim, MORL_ERR_SHAPE, "morl_dyna_commit_f32: bad shape E=%d N=%d O=%d A=%d rew_dim=%d", E,
                 N, O, A, rew_dim);
    MORL_REQUIRE(capacity > 0 && ptr >= 0 && ptr < capacity, MORL_ERR_SHAPE, "morl_dyna_commit_f32: ptr %d outside the ring of capacity %d", ptr, capacity);
    MORL_REQUIRE(rule >= MORL_TERM_NONE && rule <= MORL_TERM_LUNARLANDER, MORL_ERR_UNSUPPORTED, "morl_dyna_commit_f32: unknown termination rule %d", rule);
    const int S = O - rew_dim;
    // the columns each rule reads: s'[0] (all), s'[1] (HOPPER, MOUNTAINCAR), s'[6], s'[7] and r[0] (LUNARLANDER)
    const bool cols_ok = rule == MORL_TERM_NONE || (rule == MORL_TERM_HUMANOID && S >= 1) || ((rule == MORL_TERM_HOPPER || rule == MORL_TERM_MOUNTAINCAR) && S >= 2) ||
                         (rule == MORL_TERM_LUNARLANDER && S >= 8 && rew_dim >= 1);
    MORL_REQUIRE(cols_ok, MORL_ERR_SHAPE, "morl_dyna_commit_f32: termination rule %d reads columns that S=%d, rew_dim=%d do not have", rule, S, rew_dim);
    const int tiles = dyna_commit_tiles(N);
    int* tile_counts = static_cast<int*>(workspace);
    uint8_t* flags = reinterpret_cast<uint8_t*>(tile_counts + 2 * (size_t)tiles);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dyna_flags_kernel<<<tiles, kCommitWarps * 32, 0, s>>>(out, max_logvar, min_logvar, model_idx, noise, obs, rew_dim, E, N, O, rule, max_uncertainty,
                                                          uncertainty_out, flags, tile_counts);
    dyna_write_kernel<<<tiles, kCommitWarps * 32, 0, s>>>(out, max_logvar, min_logvar, model_idx, noise, obs, act, rew_dim, E, N, O, A, flags, tile_counts,
                                                          tiles, st_obs, st_next_obs, st_act, st_rew, st_done, capacity, ptr, next_alive, counts_out);
    return check_launch("morl_dyna_commit_f32");
}
