// nl_ppo.cu -- non-linear MO-PPO's actor-critic (reference single_policy/ser/nl_mo_ppo.py:26-108) and its minibatch update
// (nl_mo_ppo.py:325-398) on CUDA cores.
//
//   x = [obs (S) || accrued reward (d) || pref (Dp)],  Dp in {0, d}; the pref columns are one [Dp] vector shared by every row
//   critic: x -> tanh(64) -> tanh(64) -> d values,  actor: x -> tanh(64) -> tanh(64) -> A logits (Categorical)
//
// morl_nl_ppo_update_f32  : one minibatch of M rows gathered through the epoch permutation: per-objective advantage normalisation,
//                           forward of both networks, log-softmax, ratio, entropy, the per-objective clipped surrogate dotted with the
//                           loss weights w, the (clipped) vector value loss, and the backward through both networks.  A FIXED number of
//                           CTAs each folds a contiguous range of 16-row tiles, in tile order, into its own gradient and statistics
//                           partial; a second launch sums them in CTA order into the 12 .grad storages and finishes loss and stats.
// morl_nl_ppo_forward_f32 : both networks (or either) on N rows, optional first-occurrence argmax; rows and outputs may be pinned host memory
// morl_nl_ppo_commit_f32  : one rollout step's bookkeeping (nl_mo_ppo.py:251-275) for every environment in one launch
//
// The networks are tiny (hidden 64, K = S + d + Dp <= 256), so CUDA cores, activations in shared memory, no float atomics.
#include "tile_mlp.cuh"

namespace morl {

constexpr int kNlCtas = 128;    // CTAs of the update, whatever M and the card (the reduction order depends on it)
constexpr int kNlHidden = 64;   // the reference Agent's hidden width
constexpr int kNlMaxK = 256;    // S + d + Dp
constexpr int kNlMaxA = 32;
constexpr int kNlMaxBatch = 4096;
constexpr int kNlStats = MORL_MAX_D + 5;  // per CTA: pg sum per objective | value-loss sum | entropy | -logratio | kl | clipped rows

using NlParams = ParamTable<12>;
using NlGrads = GradTable<12>;
using NlLayout = ParamLayout<12>;

struct NlShape {
    int S, d, Dp, A;
    __host__ __device__ int K() const { return S + d + Dp; }
    // tensor t in the Agent's parameter order: critic W0 b0 W2 b2 W4 b4, then actor W0 b0 W2 b2 W4 b4
    NlLayout layout() const {
        NlLayout lay{12, {}};
        for (int t = 0; t < 12; ++t) {
            const int l = (t % 6) >> 1;
            const int out = l < 2 ? kNlHidden : (t < 6 ? d : A);
            const int in = l == 0 ? K() : kNlHidden;
            lay.size[t] = (t & 1) ? out : out * in;
        }
        return lay;
    }
};

// The activations of one tile in shared memory: input, both networks' hidden layers, outputs, and the backward's two buffers.
struct NlTile {
    float x[kTileRows * kNlMaxK];
    float h1[2][kTileRows * kNlHidden];  // [0] critic, [1] actor
    float h2[2][kTileRows * kNlHidden];
    float z[kTileRows * kNlMaxA];        // logits, then d loss / d logits
    float v[kTileRows * MORL_MAX_D];     // values, then d loss / d values
    float dh[2][kTileRows * kNlHidden];
};

// Network `net` (0 critic, 1 actor) on the staged tile; its outputs go to `out` [kTileRows, N].
__device__ void nl_forward(const NlParams& P, const NlShape& sh, NlTile& m, int net, float* out, int N) {
    const float* const* p = P.p + 6 * net;
    tile_linear(p[0], p[1], m.x, sh.K(), m.h1[net], kNlHidden, Act::Tanh);
    tile_linear(p[2], p[3], m.h1[net], kNlHidden, m.h2[net], kNlHidden, Act::Tanh);
    tile_linear(p[4], p[5], m.h2[net], kNlHidden, out, N, Act::None);
}

// Backward of network `net` from d loss / d outputs `dz` [kTileRows, N] (the tile's forward activations still in place).
__device__ void nl_backward(const NlParams& P, const NlShape& sh, const NlLayout& lay, NlTile& m, int net, const float* dz, int N, float* g,
                            bool init) {
    const int t0 = 6 * net;
    tile_backward(P.p[t0 + 4], m.h2[net], kNlHidden, dz, N, g + lay.offset(t0 + 4), g + lay.offset(t0 + 5), init, m.dh[0], Act::Tanh);
    tile_backward(P.p[t0 + 2], m.h1[net], kNlHidden, m.dh[0], kNlHidden, g + lay.offset(t0 + 2), g + lay.offset(t0 + 3), init, m.dh[1], Act::Tanh);
    tile_backward(P.p[t0 + 0], m.x, sh.K(), m.dh[1], kNlHidden, g + lay.offset(t0 + 0), g + lay.offset(t0 + 1), init, nullptr, Act::Tanh);
}

// Stages rows [r0, r0 + kTileRows) as x = [obs || acc || pref], zero past n.  Row r reads source row src(r).
template <typename Src>
__device__ __forceinline__ void nl_stage(NlTile& m, const NlShape& sh, const float* obs, const float* acc, const float* __restrict__ pref, int r0,
                                         int n, Src src) {
    const int K = sh.K(), S = sh.S, d = sh.d;
    for (int idx = threadIdx.x; idx < kTileRows * K; idx += kTileThreads) {
        const int r = idx / K, k = idx % K, row = r0 + r;
        float v = 0.f;
        if (row < n) {
            const size_t s = src(row);
            v = k < S ? obs[s * S + k] : (k < S + d ? acc[s * d + (k - S)] : __ldg(pref + (k - S - d)));
        }
        m.x[idx] = v;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kTileThreads) nl_update_kernel(
    const __grid_constant__ NlParams P, const __grid_constant__ NlShape sh, const __grid_constant__ NlLayout lay, const float* __restrict__ obs, const float* __restrict__ acc,
    const int64_t* __restrict__ actions, const float* __restrict__ old_logp, const float* __restrict__ adv, const float* __restrict__ ret,
    const float* __restrict__ old_v, const int64_t* __restrict__ perm, int M, const float* __restrict__ pref, const float* __restrict__ w,
    float clip_coef, float ent_coef, float vf_coef, int norm_adv, int clip_vloss, float* __restrict__ part, double* __restrict__ stat_part) {
    __shared__ NlTile m;
    __shared__ double red[kTileWarps];
    __shared__ double red_lane[kTileWarps][32];
    __shared__ float s_mu[MORL_MAX_D], s_den[MORL_MAX_D], s_w[MORL_MAX_D];
    const int d = sh.d, A = sh.A;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // per-objective advantage mean and unbiased std of the whole minibatch (every CTA computes the same values, in the same order)
    if (threadIdx.x < d) {
        s_mu[threadIdx.x] = 0.f;
        s_den[threadIdx.x] = 1.f;
        s_w[threadIdx.x] = __ldg(w + threadIdx.x);
    }
    if (norm_adv) {
        for (int o = 0; o < d; ++o) {
            double s = 0.0;
            for (int i = threadIdx.x; i < M; i += kTileThreads) s += (double)__ldg(adv + (size_t)__ldg(perm + i) * d + o);
            const double mean = block_sum_f64<kTileThreads>(s, red) / (double)M;
            double s2 = 0.0;
            for (int i = threadIdx.x; i < M; i += kTileThreads) {
                const double c = (double)__ldg(adv + (size_t)__ldg(perm + i) * d + o) - mean;
                s2 += c * c;
            }
            const double var = block_sum_f64<kTileThreads>(s2, red) / (double)(M - 1);
            if (threadIdx.x == 0) {
                s_mu[o] = (float)mean;
                s_den[o] = __fadd_rn((float)sqrt(var), 1e-8f);
            }
        }
    }
    __syncthreads();

    const int c = blockIdx.x;
    int first, count;
    tile_range((M + kTileRows - 1) / kTileRows, c, first, count);
    float* out = part + (size_t)c * lay.total();
    const float inv_m = 1.0f / (float)M;
    const float g_v = (float)(0.5 / ((double)M * d)) * vf_coef;
    const float g_ent = __fmul_rn(ent_coef, inv_m);
    const float lo = __fsub_rn(1.0f, clip_coef), hi = __fadd_rn(1.0f, clip_coef);
    double pg_acc = 0.0, v_acc = 0.0;                          // lane o: objective o
    double ent_acc = 0.0, okl_acc = 0.0, kl_acc = 0.0, clip_acc = 0.0;  // lane 0

    for (int tile = first; tile < first + count; ++tile) {
        const bool init = tile == first;
        const int r0 = tile * kTileRows;
        nl_stage(m, sh, obs, acc, pref, r0, M, [&](int row) { return (size_t)__ldg(perm + row); });
        nl_forward(P, sh, m, 0, m.v, d);
        nl_forward(P, sh, m, 1, m.z, A);

        // one warp per row; lane a holds logit a, lane o objective o
        for (int r = warp; r < kTileRows; r += kTileWarps) {
            const int row = r0 + r;
            const bool valid = row < M;
            const size_t src = valid ? (size_t)__ldg(perm + row) : 0;
            const float z = lane < A ? m.z[r * A + lane] : -INFINITY;
            const float mx = warp_max_f32(z);
            const float e = lane < A ? expf(__fsub_rn(z, mx)) : 0.f;
            const float lse = __fadd_rn(logf(warp_sum_f32(e)), mx);
            const float l = __fsub_rn(z, lse);  // log-probability of action `lane`
            const float p = lane < A ? expf(l) : 0.f;
            const float ent = -warp_sum_f32(lane < A ? __fmul_rn(l, p) : 0.f);
            const int a = valid ? (int)__ldg(actions + src) : 0;
            const float logratio = __fsub_rn(__shfl_sync(0xffffffffu, l, a & 31), valid ? __ldg(old_logp + src) : 0.f);
            const float ratio = expf(logratio);
            // per-objective clipped surrogate and the gradient it sends to the ratio (th.max splits a tie; clamp passes on [lo, hi])
            float dratio_o = 0.f, dv = 0.f;
            if (valid && lane < d) {
                float av = __ldg(adv + src * d + lane);
                av = __fdiv_rn(__fsub_rn(av, s_mu[lane]), s_den[lane]);
                const float rc = fminf(fmaxf(ratio, lo), hi);
                const float pg1 = __fmul_rn(-av, ratio), pg2 = __fmul_rn(-av, rc);
                pg_acc += (double)fmaxf(pg1, pg2);
                const float w1 = pg1 > pg2 ? 1.0f : (pg1 == pg2 ? 0.5f : 0.0f);
                const float in_band = (ratio >= lo && ratio <= hi) ? 1.0f : 0.0f;
                dratio_o = __fmul_rn(__fmul_rn(s_w[lane], inv_m), __fmul_rn(-av, __fadd_rn(w1, __fmul_rn(1.0f - w1, in_band))));
                const float nv = m.v[r * d + lane], R = __ldg(ret + src * d + lane);
                const float du = __fsub_rn(nv, R);
                const float vu = __fmul_rn(du, du);
                float g;
                if (clip_vloss) {
                    const float ov = __ldg(old_v + src * d + lane);
                    const float dd = __fsub_rn(nv, ov);
                    const float dc = __fsub_rn(__fadd_rn(ov, fminf(fmaxf(dd, -clip_coef), clip_coef)), R);
                    const float vc = __fmul_rn(dc, dc);
                    v_acc += (double)fmaxf(vu, vc);
                    const float u1 = vu > vc ? 1.0f : (vu == vc ? 0.5f : 0.0f);
                    const float band = (dd >= -clip_coef && dd <= clip_coef) ? 1.0f : 0.0f;
                    g = __fadd_rn(__fmul_rn(u1, __fmul_rn(2.0f, du)), __fmul_rn(__fmul_rn(1.0f - u1, band), __fmul_rn(2.0f, dc)));
                } else {
                    v_acc += (double)vu;
                    g = __fmul_rn(2.0f, du);
                }
                dv = __fmul_rn(g_v, g);
            }
            const float dlp = __fmul_rn(warp_sum_f32(dratio_o), ratio);  // d loss / d log p_a
            if (valid && lane == 0) {
                ent_acc += (double)ent;
                okl_acc += (double)(-logratio);
                kl_acc += (double)__fsub_rn(__fsub_rn(ratio, 1.0f), logratio);
                clip_acc += (fabsf(__fsub_rn(ratio, 1.0f)) > clip_coef) ? 1.0 : 0.0;
            }
            // d loss / d z_k = dlp ([k == a] - p_k) - (ent_coef / M) dH/dz_k,  dH/dz_k = -p_k (l_k + H)
            if (lane < A)
                m.z[r * A + lane] = valid ? __fadd_rn(__fmul_rn(dlp, __fsub_rn(lane == a ? 1.0f : 0.0f, p)), __fmul_rn(g_ent, __fmul_rn(p, __fadd_rn(l, ent))))
                                          : 0.f;
            if (lane < d) m.v[r * d + lane] = dv;
        }
        __syncthreads();
        nl_backward(P, sh, lay, m, 1, m.z, A, out, init);
        nl_backward(P, sh, lay, m, 0, m.v, d, out, init);
    }

    // statistics partial of this CTA, summed over its warps in order
    red_lane[warp][lane] = pg_acc;
    __syncthreads();
    double* sp = stat_part + (size_t)c * kNlStats;
    if (threadIdx.x < d) {
        double t = 0.0;
        for (int i = 0; i < kTileWarps; ++i) t += red_lane[i][threadIdx.x];
        sp[threadIdx.x] = t;
    }
    const double vs = block_sum_f64<kTileThreads>(v_acc, red);
    const double es = block_sum_f64<kTileThreads>(ent_acc, red);
    const double os = block_sum_f64<kTileThreads>(okl_acc, red);
    const double ks = block_sum_f64<kTileThreads>(kl_acc, red);
    const double cs = block_sum_f64<kTileThreads>(clip_acc, red);
    if (threadIdx.x == 0) {
        sp[MORL_MAX_D + 0] = vs;
        sp[MORL_MAX_D + 1] = es;
        sp[MORL_MAX_D + 2] = os;
        sp[MORL_MAX_D + 3] = ks;
        sp[MORL_MAX_D + 4] = cs;
    }
}

// Block 0 of the partial sum: the loss and the statistics from the CTAs' statistics partials.
struct NlFinish {
    const double* stat_part;
    int M, d;
    const float* w;
    float ent_coef, vf_coef;
    float* loss_out;
    float* stats;
    __device__ void operator()(int n_parts) const {
        __shared__ double acc[kNlStats];
        if (threadIdx.x < kNlStats) {
            double t = 0.0;
            for (int c = 0; c < n_parts; ++c) t += stat_part[(size_t)c * kNlStats + threadIdx.x];
            acc[threadIdx.x] = t;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const double inv_m = 1.0 / (double)M;
            float pg = 0.f;  // (per-objective mean surrogate * w).sum()
            for (int o = 0; o < d; ++o) pg = __fadd_rn(pg, __fmul_rn((float)(acc[o] * inv_m), __ldg(w + o)));
            const float v = (float)(0.5 * acc[MORL_MAX_D] / ((double)M * d));
            const float ent = (float)(acc[MORL_MAX_D + 1] * inv_m);
            if (loss_out) loss_out[0] = __fadd_rn(__fsub_rn(pg, __fmul_rn(ent_coef, ent)), __fmul_rn(vf_coef, v));
            stats[0] = pg;
            stats[1] = v;
            stats[2] = ent;
            stats[3] = (float)(acc[MORL_MAX_D + 2] * inv_m);
            stats[4] = (float)(acc[MORL_MAX_D + 3] * inv_m);
            stats[5] = __fadd_rn(stats[5], (float)(acc[MORL_MAX_D + 4] * inv_m));
        }
    }
};

// Both networks (as asked) on N rows [obs || acc || pref]; obs, acc and the outputs may live in mapped pinned host memory.
__global__ void __launch_bounds__(kTileThreads) nl_forward_kernel(const __grid_constant__ NlParams P, const __grid_constant__ NlShape sh,
                                                                const float* obs, const float* acc, const float* __restrict__ pref, int N,
                                                                float* logits, float* values, int32_t* argmax) {
    __shared__ NlTile m;
    const int r0 = blockIdx.x * kTileRows;
    const int nr = min(kTileRows, N - r0);
    const int d = sh.d, A = sh.A;
    nl_stage(m, sh, obs, acc, pref, r0, N, [](int row) { return (size_t)row; });
    if (values) {
        nl_forward(P, sh, m, 0, m.v, d);
        for (int idx = threadIdx.x; idx < nr * d; idx += kTileThreads) values[(size_t)r0 * d + idx] = m.v[idx];
    }
    if (logits || argmax) {
        nl_forward(P, sh, m, 1, m.z, A);
        for (int idx = threadIdx.x; logits && idx < nr * A; idx += kTileThreads) logits[(size_t)r0 * A + idx] = m.z[idx];
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int r = warp; argmax && r < nr; r += kTileWarps) {
            // first occurrence of the row maximum (torch.argmax)
            float best = lane < A ? m.z[r * A + lane] : -INFINITY;
            int bi = lane < A ? lane : kNlMaxA;
            warp_argmax(best, bi);
            if (lane == 0) argmax[r0 + r] = bi;
        }
    }
}

// One rollout step for environment e (one thread each).  The carried state (next_obs, next_acc, next_done, timestep) is stored into row
// `step` of the rollout, then replaced by the environment's outputs staged as [obs (S) | reward (d) | terminated | truncated] per env:
//   acc' = (acc + gamma^t * r) * (1 - done),  t' = (t + 1) * (1 - done),  done = terminated | truncated   (nl_mo_ppo.py:251-275)
__global__ void nl_commit_kernel(const float* __restrict__ staged, const float* __restrict__ logits, const int64_t* __restrict__ action, int step,
                                 int E, int S, int d, int A, float gamma, float* __restrict__ obs_store, float* __restrict__ acc_store,
                                 float* __restrict__ done_store, float* __restrict__ rew_store, int64_t* __restrict__ act_store,
                                 float* __restrict__ logp_store, float* __restrict__ next_obs, float* __restrict__ next_acc,
                                 float* __restrict__ next_done, int32_t* __restrict__ timestep) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const size_t row = (size_t)step * E + e;
    const float* in = staged + (size_t)e * (S + d + 2);
    for (int k = 0; k < S; ++k) {
        obs_store[row * S + k] = next_obs[(size_t)e * S + k];
        next_obs[(size_t)e * S + k] = in[k];
    }
    done_store[row] = next_done[e];
    const float done = (in[S + d] != 0.f || in[S + d + 1] != 0.f) ? 1.0f : 0.0f;
    next_done[e] = done;
    const int t = timestep[e];
    const float gt = powf(gamma, (float)t);  // torch's device pow of (float scalar) ** (int32 tensor), computed in float32
    const float keep = __fsub_rn(1.0f, done);
    for (int o = 0; o < d; ++o) {
        const float r = in[S + o];
        const float a0 = next_acc[(size_t)e * d + o];
        acc_store[row * d + o] = a0;
        rew_store[row * d + o] = r;
        next_acc[(size_t)e * d + o] = __fmul_rn(__fadd_rn(a0, __fmul_rn(gt, r)), keep);
    }
    timestep[e] = (t + 1) * (1 - (int)done);
    // log-probability of the sampled action: z_a - (log sum exp(z - max) + max)
    const float* z = logits + (size_t)e * A;
    float mx = -INFINITY;
    for (int j = 0; j < A; ++j) mx = fmaxf(mx, z[j]);
    float s = 0.f;
    for (int j = 0; j < A; ++j) s = __fadd_rn(s, expf(__fsub_rn(z[j], mx)));
    const int64_t a = action[e];
    act_store[row] = a;
    logp_store[row] = __fsub_rn(z[a], __fadd_rn(logf(s), mx));
}

static bool nl_shape(int obs_dim, int d, int pref_dim, int n_actions, NlShape* sh) {
    if (obs_dim < 1 || d < 1 || d > MORL_MAX_D || (pref_dim != 0 && pref_dim != d) || obs_dim + d + pref_dim > kNlMaxK || n_actions < 1 ||
        n_actions > kNlMaxA)
        return false;
    sh->S = obs_dim;
    sh->d = d;
    sh->Dp = pref_dim;
    sh->A = n_actions;
    return true;
}

}  // namespace morl

extern "C" int morl_nl_ppo_supported(int obs_dim, int d, int pref_dim, int n_actions, int batch) {
    morl::NlShape sh;
    return morl::nl_shape(obs_dim, d, pref_dim, n_actions, &sh) && batch >= 1 && batch <= morl::kNlMaxBatch ? 1 : 0;
}

extern "C" size_t morl_nl_ppo_workspace_bytes(int obs_dim, int d, int pref_dim, int n_actions) {
    using namespace morl;
    NlShape sh;
    if (!nl_shape(obs_dim, d, pref_dim, n_actions, &sh)) return 0;
    return (size_t)kNlCtas * kNlStats * sizeof(double) + (size_t)kNlCtas * (size_t)sh.layout().total() * sizeof(float);
}

extern "C" int morl_nl_ppo_update_f32(const float* const* params, float* const* grads, const float* obs, const float* acc, const int64_t* actions,
                                      const float* old_logprob, const float* advantages, const float* returns, const float* old_values,
                                      const int64_t* perm, int M, int obs_dim, int d, int pref_dim, int n_actions, const float* pref,
                                      const float* loss_weights, float clip_coef, float ent_coef, float vf_coef, int norm_adv, int clip_vloss,
                                      float* loss_out, float* stats, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && grads && obs && acc && actions && old_logprob && advantages && returns && perm && loss_weights && stats && workspace,
                 MORL_ERR_NULL, "morl_nl_ppo_update_f32: NULL pointer argument");
    MORL_REQUIRE(!clip_vloss || old_values, MORL_ERR_NULL, "morl_nl_ppo_update_f32: clip_vloss needs old_values");
    MORL_REQUIRE(pref_dim == 0 || pref, MORL_ERR_NULL, "morl_nl_ppo_update_f32: pref_dim=%d needs pref", pref_dim);
    NlShape sh;
    MORL_REQUIRE(morl_nl_ppo_supported(obs_dim, d, pref_dim, n_actions, M) && nl_shape(obs_dim, d, pref_dim, n_actions, &sh), MORL_ERR_UNSUPPORTED,
                 "morl_nl_ppo_update_f32: unsupported configuration S=%d d=%d Dp=%d A=%d M=%d (morl_nl_ppo_supported)", obs_dim, d, pref_dim,
                 n_actions, M);
    MORL_REQUIRE(!norm_adv || M >= 2, MORL_ERR_SHAPE, "morl_nl_ppo_update_f32: advantage normalisation needs M >= 2 rows (unbiased std), got M=%d", M);
    NlParams P;
    NlGrads G;
    if (int rc = load_tables("morl_nl_ppo_update_f32", 12, params, P, grads, &G)) return rc;
    const NlLayout lay = sh.layout();
    const int ctas = min(kNlCtas, (M + kTileRows - 1) / kTileRows);
    double* stat_part = static_cast<double*>(workspace);
    float* part = reinterpret_cast<float*>(stat_part + (size_t)kNlCtas * kNlStats);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    nl_update_kernel<<<ctas, kTileThreads, 0, st>>>(P, sh, lay, obs, acc, actions, old_logprob, advantages, returns, old_values, perm, M, pref, loss_weights,
                                                  clip_coef, ent_coef, vf_coef, norm_adv ? 1 : 0, clip_vloss ? 1 : 0, part, stat_part);
    launch_partial_sum(G, lay, part, ctas, NlFinish{stat_part, M, d, loss_weights, ent_coef, vf_coef, loss_out, stats}, st);
    return check_launch("morl_nl_ppo_update_f32");
}

extern "C" int morl_nl_ppo_forward_f32(const float* const* params, const float* obs, const float* acc, int N, int obs_dim, int d, int pref_dim,
                                       int n_actions, const float* pref, float* logits, float* values, int32_t* argmax_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && obs && acc && (logits || values || argmax_out), MORL_ERR_NULL, "morl_nl_ppo_forward_f32: NULL pointer argument");
    MORL_REQUIRE(pref_dim == 0 || pref, MORL_ERR_NULL, "morl_nl_ppo_forward_f32: pref_dim=%d needs pref", pref_dim);
    MORL_REQUIRE(N > 0, MORL_ERR_SHAPE, "morl_nl_ppo_forward_f32: bad shape N=%d", N);
    NlShape sh;
    MORL_REQUIRE(nl_shape(obs_dim, d, pref_dim, n_actions, &sh), MORL_ERR_UNSUPPORTED,
                 "morl_nl_ppo_forward_f32: unsupported configuration S=%d d=%d Dp=%d A=%d (morl_nl_ppo_supported)", obs_dim, d, pref_dim, n_actions);
    NlParams P;
    if (int rc = load_tables("morl_nl_ppo_forward_f32", 12, params, P)) return rc;
    nl_forward_kernel<<<(N + kTileRows - 1) / kTileRows, kTileThreads, 0, static_cast<cudaStream_t>(stream)>>>(P, sh, obs, acc, pref, N, logits, values,
                                                                                                         argmax_out);
    return check_launch("morl_nl_ppo_forward_f32");
}

extern "C" int morl_nl_ppo_commit_f32(const float* staged, const float* logits, const int64_t* action, int step, int E, int obs_dim, int d,
                                      int n_actions, double gamma, float* obs_store, float* acc_store, float* done_store, float* rew_store,
                                      int64_t* act_store, float* logp_store, float* next_obs, float* next_acc, float* next_done, int32_t* timestep,
                                      void* stream) {
    using namespace morl;
    MORL_REQUIRE(staged && logits && action && obs_store && acc_store && done_store && rew_store && act_store && logp_store && next_obs && next_acc &&
                     next_done && timestep,
                 MORL_ERR_NULL, "morl_nl_ppo_commit_f32: NULL pointer argument");
    MORL_REQUIRE(E > 0 && obs_dim > 0 && d > 0 && n_actions > 0 && step >= 0, MORL_ERR_SHAPE,
                 "morl_nl_ppo_commit_f32: bad shape E=%d S=%d d=%d A=%d step=%d", E, obs_dim, d, n_actions, step);
    constexpr int kThreads = 128;
    nl_commit_kernel<<<(E + kThreads - 1) / kThreads, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        staged, logits, action, step, E, obs_dim, d, n_actions, (float)gamma, obs_store, acc_store, done_store, rew_store, act_store, logp_store,
        next_obs, next_acc, next_done, timestep);
    return check_launch("morl_nl_ppo_commit_f32");
}
