// ppo.cu -- the device side of MO-PPO's update (reference single_policy/ser/mo_ppo.py).
//
// morl_vector_gae_f32            : the reverse GAE / discounted-return recursion of :439-476 in one launch
// morl_vector_gae_objectives_f32 : the same recursion, keeping the per-objective advantages (nl_mo_ppo.py:290-308)
// morl_ppo_loss_f32   : one minibatch's clipped PPO loss, its gradients w.r.t. the actor mean, actor_logstd and the vector value head,
//                       and the logged statistics (:514-549) in one launch
#include "common.cuh"

namespace morl {

// ---- vector GAE ------------------------------------------------------------------------------------------------------------------
// One lane per (env, objective), sequential over T from the last step back.  A CTA owns 32 / d whole environments, so the
// scalarisation of its advantages needs no other CTA.  Chunks of kGaeChunk steps of rewards, values and dones are staged in shared
// memory by the whole CTA before the lanes walk them, so the dependent chain never waits on a global load.  kScalarise = false writes
// each lane's advantage to adv_out [T, E, D] as it is produced and skips the scalarisation.
constexpr int kGaeThreads = 128;
constexpr int kGaeLanes = 32;  // (env, objective) lanes per CTA; the lanes of one env are never split
constexpr int kGaeChunk = 64;

template <bool kScalarise>
__global__ void __launch_bounds__(kGaeThreads) vector_gae_kernel(const float* __restrict__ rewards, const float* __restrict__ values,
                                                                 const float* __restrict__ dones, const float* __restrict__ next_value,
                                                                 const float* __restrict__ next_done, const float* __restrict__ w, int T, int E,
                                                                 int D, int envs_per_cta, float gamma, float gl, int use_gae,
                                                                 float* __restrict__ returns, float* __restrict__ adv_out) {
    __shared__ float s_r[kGaeChunk][kGaeLanes];
    __shared__ float s_v[kGaeChunk][kGaeLanes];
    __shared__ float s_a[kGaeChunk][kGaeLanes];  // per-objective advantages of the chunk, scalarised after the walk
    __shared__ float s_nd[kGaeChunk + 1][kGaeLanes];  // 1 - done of the chunk's steps and of the step after it
    const int e0 = blockIdx.x * envs_per_cta;
    const int ne = min(envs_per_cta, E - e0);
    const int nl = ne * D;  // active lanes
    const size_t row = (size_t)E * D;
    const int lane = threadIdx.x;
    float carry = 0.f;  // GAE: lastgaelam (0 before the last step);  plain returns: next_return
    float nv = 0.f;     // GAE: value of the step after the current one
    if (lane < nl) {
        nv = __ldg(next_value + (size_t)e0 * D + lane);
        if (!use_gae) carry = nv;
    }
    for (int t1 = T; t1 > 0; t1 -= kGaeChunk) {
        const int t0 = max(0, t1 - kGaeChunk);
        const int n = t1 - t0;
        __syncthreads();  // the previous chunk's scalarisation has read s_a
        for (int k = threadIdx.x; k < n * nl; k += blockDim.x) {
            const int tt = k / nl, l = k - tt * nl;
            const size_t g = (size_t)(t0 + tt) * row + (size_t)e0 * D + l;
            s_r[tt][l] = __ldg(rewards + g);
            s_v[tt][l] = __ldg(values + g);
        }
        for (int k = threadIdx.x; k < (n + 1) * ne; k += blockDim.x) {
            const int tt = k / ne, e = k - tt * ne;
            const int t = t0 + tt;  // dones of step t + 1 feed step t; t == T is next_done
            const float dn = (t < T) ? __ldg(dones + (size_t)t * E + e0 + e) : __ldg(next_done + e0 + e);
            s_nd[tt][e] = __fsub_rn(1.0f, dn);
        }
        __syncthreads();
        if (lane < nl) {
            const int e = lane / D;
            for (int tt = n - 1; tt >= 0; --tt) {
                const float nnt = s_nd[tt + 1][e];
                const float r = s_r[tt][lane], v = s_v[tt][lane];
                float a;
                if (use_gae) {
                    // delta = r + gamma * nextvalues * nnt - v;  lastgaelam = delta + (gamma * lambda) * nnt * lastgaelam
                    const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(__fmul_rn(gamma, nv), nnt)), v);
                    carry = __fadd_rn(delta, __fmul_rn(__fmul_rn(gl, nnt), carry));
                    a = carry;
                    returns[(size_t)(t0 + tt) * row + (size_t)e0 * D + lane] = __fadd_rn(a, v);
                    nv = v;
                } else {
                    // returns[t] = r + gamma * nnt * next_return;  advantages = returns - values
                    carry = __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, nnt), carry));
                    returns[(size_t)(t0 + tt) * row + (size_t)e0 * D + lane] = carry;
                    a = __fsub_rn(carry, v);
                }
                if constexpr (kScalarise)
                    s_a[tt][lane] = a;
                else
                    adv_out[(size_t)(t0 + tt) * row + (size_t)e0 * D + lane] = a;
            }
        }
        if constexpr (!kScalarise) continue;
        __syncthreads();
        for (int k = threadIdx.x; k < n * ne; k += blockDim.x) {
            const int tt = k / ne, e = k - tt * ne;
            double s = 0.0;  // the d-term dot product, summed exactly enough to be rounded once
            for (int o = 0; o < D; ++o) s += (double)s_a[tt][e * D + o] * (double)__ldg(w + o);
            adv_out[(size_t)(t0 + tt) * E + e0 + e] = (float)s;
        }
    }
}

// ---- PPO loss --------------------------------------------------------------------------------------------------------------------
// One CTA walks the M rows three times (row statistics, the unbiased std of the advantages, then the loss terms and gradients).  Every
// reduction is a fixed-shape block tree in double, so the result does not depend on scheduling.
constexpr int kPpoThreads = 256;
constexpr int kPpoMaxA = 32;
constexpr float kHalfLog2Pi = 0.918938533204672742f;  // 0.5 * log(2 pi)

// Normal(mean, exp(logstd)).log_prob(action).sum(-1) for one row
__device__ __forceinline__ float row_logprob(const float* __restrict__ mean, const float* __restrict__ act, const float* s_ls,
                                             const float* s_ivar, int A) {
    float lp = 0.f;
    for (int j = 0; j < A; ++j) {
        const float z = __fsub_rn(__ldg(act + j), __ldg(mean + j));
        lp = __fadd_rn(lp, __fsub_rn(__fsub_rn(-__fmul_rn(__fmul_rn(z, z), 0.5f * s_ivar[j]), s_ls[j]), kHalfLog2Pi));
    }
    return lp;
}

__global__ void __launch_bounds__(kPpoThreads) ppo_loss_kernel(const float* __restrict__ mean, const float* __restrict__ logstd,
                                                               const float* __restrict__ value, const float* __restrict__ actions,
                                                               const float* __restrict__ old_logprob, const float* __restrict__ advantages,
                                                               const float* __restrict__ returns, const float* __restrict__ old_values, int M,
                                                               int A, int D, float clip_coef, float ent_coef, float vf_coef, int norm_adv,
                                                               int clip_vloss, float* __restrict__ loss_out, float* __restrict__ dmean,
                                                               float* __restrict__ dlogstd, float* __restrict__ dvalue, float* __restrict__ stats) {
    __shared__ double red[kPpoThreads / 32];
    __shared__ float s_ls[kPpoMaxA], s_ivar[kPpoMaxA];
    if (threadIdx.x < A) {
        const float ls = __ldg(logstd + threadIdx.x);
        const float sd = expf(ls);
        s_ls[threadIdx.x] = ls;
        s_ivar[threadIdx.x] = __frcp_rn(__fmul_rn(sd, sd));
    }
    __syncthreads();
    const double inv_m = 1.0 / (double)M;

    // pass 1: advantage mean, KL estimates, clip fraction
    double s_adv = 0.0, s_okl = 0.0, s_kl = 0.0, s_clip = 0.0;
    for (int i = threadIdx.x; i < M; i += kPpoThreads) {
        const float lr = __fsub_rn(row_logprob(mean + (size_t)i * A, actions + (size_t)i * A, s_ls, s_ivar, A), __ldg(old_logprob + i));
        const float ratio = expf(lr);
        s_adv += (double)__ldg(advantages + i);
        s_okl += (double)(-lr);
        s_kl += (double)__fsub_rn(__fsub_rn(ratio, 1.0f), lr);
        s_clip += (fabsf(__fsub_rn(ratio, 1.0f)) > clip_coef) ? 1.0 : 0.0;
    }
    const double adv_mean = block_sum_f64<kPpoThreads>(s_adv, red) * inv_m;
    const double okl = block_sum_f64<kPpoThreads>(s_okl, red) * inv_m;
    const double kl = block_sum_f64<kPpoThreads>(s_kl, red) * inv_m;
    const double clipfrac = block_sum_f64<kPpoThreads>(s_clip, red) * inv_m;

    // pass 2: unbiased standard deviation (torch's Tensor.std())
    float a_mu = 0.f, a_den = 1.f;
    if (norm_adv) {
        double s2 = 0.0;
        for (int i = threadIdx.x; i < M; i += kPpoThreads) {
            const double c = (double)__ldg(advantages + i) - adv_mean;
            s2 += c * c;
        }
        const double var = block_sum_f64<kPpoThreads>(s2, red) / (double)(M - 1);
        a_mu = (float)adv_mean;
        a_den = __fadd_rn((float)sqrt(var), 1e-8f);
    }

    // pass 3: policy and value losses and their gradients
    const float lo = __fsub_rn(1.0f, clip_coef), hi = __fadd_rn(1.0f, clip_coef);
    const float g_pg = (float)inv_m;
    const float g_v = (float)(0.5 / ((double)M * D)) * vf_coef;
    double s_pg = 0.0, s_v = 0.0;
    double acc[kPpoMaxA];
#pragma unroll
    for (int j = 0; j < kPpoMaxA; ++j) acc[j] = 0.0;
    for (int i = threadIdx.x; i < M; i += kPpoThreads) {
        const float* mu = mean + (size_t)i * A;
        const float* act = actions + (size_t)i * A;
        const float lr = __fsub_rn(row_logprob(mu, act, s_ls, s_ivar, A), __ldg(old_logprob + i));
        const float ratio = expf(lr);
        float adv = __ldg(advantages + i);
        if (norm_adv) adv = __fdiv_rn(__fsub_rn(adv, a_mu), a_den);
        const float rc = fminf(fmaxf(ratio, lo), hi);
        const float pg1 = __fmul_rn(-adv, ratio), pg2 = __fmul_rn(-adv, rc);
        s_pg += (double)fmaxf(pg1, pg2);
        // th.max backward: the larger operand takes the gradient, a tie splits it; clamp passes it on its closed interval
        const float w1 = pg1 > pg2 ? 1.0f : (pg1 == pg2 ? 0.5f : 0.0f);
        const float w2 = 1.0f - w1;
        const float in_band = (ratio >= lo && ratio <= hi) ? 1.0f : 0.0f;
        const float dratio = __fmul_rn(g_pg, __fmul_rn(-adv, __fadd_rn(w1, __fmul_rn(w2, in_band))));
        const float dlp = __fmul_rn(dratio, ratio);  // d ratio / d logprob = ratio
        float* dm = dmean + (size_t)i * A;
#pragma unroll
        for (int j = 0; j < kPpoMaxA; ++j) {
            if (j < A) {
                const float z = __fsub_rn(__ldg(act + j), __ldg(mu + j));
                const float zi = __fmul_rn(z, s_ivar[j]);
                dm[j] = __fmul_rn(dlp, zi);
                acc[j] += (double)dlp * (double)__fsub_rn(__fmul_rn(zi, z), 1.0f);
            }
        }
        for (int o = 0; o < D; ++o) {
            const size_t k = (size_t)i * D + o;
            const float nv = __ldg(value + k), R = __ldg(returns + k);
            const float du = __fsub_rn(nv, R);
            const float vu = __fmul_rn(du, du);
            float g;
            if (clip_vloss) {
                const float ov = __ldg(old_values + k);
                const float dd = __fsub_rn(nv, ov);
                const float dc = __fsub_rn(__fadd_rn(ov, fminf(fmaxf(dd, -clip_coef), clip_coef)), R);
                const float vc = __fmul_rn(dc, dc);
                s_v += (double)fmaxf(vu, vc);
                const float u1 = vu > vc ? 1.0f : (vu == vc ? 0.5f : 0.0f);
                const float band = (dd >= -clip_coef && dd <= clip_coef) ? 1.0f : 0.0f;
                g = __fadd_rn(__fmul_rn(u1, __fmul_rn(2.0f, du)), __fmul_rn(__fmul_rn(1.0f - u1, band), __fmul_rn(2.0f, dc)));
            } else {
                s_v += (double)vu;
                g = __fmul_rn(2.0f, du);
            }
            dvalue[k] = __fmul_rn(g_v, g);
        }
    }
    const float pg_loss = (float)(block_sum_f64<kPpoThreads>(s_pg, red) * inv_m);
    const float v_loss = (float)(0.5 * block_sum_f64<kPpoThreads>(s_v, red) / ((double)M * D));
    // Normal entropy summed over action dims (the same for every row): sum_j 0.5 + 0.5 log(2 pi) + logstd_j
    float ent = 0.f;
    for (int j = 0; j < A; ++j) ent = __fadd_rn(ent, __fadd_rn(0.5f + kHalfLog2Pi, s_ls[j]));
#pragma unroll
    for (int j = 0; j < kPpoMaxA; ++j) {
        if (j < A) {  // uniform across the CTA
            const double sj = block_sum_f64<kPpoThreads>(acc[j], red);
            if (threadIdx.x == 0) dlogstd[j] = __fsub_rn((float)sj, ent_coef);
        }
    }
    if (threadIdx.x == 0) {
        loss_out[0] = __fadd_rn(__fsub_rn(pg_loss, __fmul_rn(ent_coef, ent)), __fmul_rn(v_loss, vf_coef));
        stats[0] = pg_loss;
        stats[1] = v_loss;
        stats[2] = ent;
        stats[3] = (float)okl;
        stats[4] = (float)kl;
        stats[5] = __fadd_rn(stats[5], (float)clipfrac);
    }
}

}  // namespace morl

extern "C" int morl_vector_gae_f32(const float* rewards, const float* values, const float* dones, const float* next_value, const float* next_done,
                                   const float* weights, int T, int E, int D, double gamma, double gae_lambda, int use_gae, float* returns,
                                   float* advantages, void* stream) {
    using namespace morl;
    MORL_REQUIRE(rewards && values && dones && next_value && next_done && weights && returns && advantages, MORL_ERR_NULL,
                 "morl_vector_gae_f32: NULL pointer argument");
    MORL_REQUIRE(T > 0 && E > 0 && D > 0, MORL_ERR_SHAPE, "morl_vector_gae_f32: bad shape T=%d E=%d D=%d", T, E, D);
    MORL_REQUIRE(D <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "morl_vector_gae_f32: D=%d > %d", D, MORL_MAX_D);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int envs_per_cta = kGaeLanes / D;
    const int blocks = (E + envs_per_cta - 1) / envs_per_cta;
    // gamma and gamma * lambda are Python floats in the reference: gamma is rounded to fp32 by the tensor op, gamma * lambda is formed
    // in double and rounded once
    vector_gae_kernel<true><<<blocks, kGaeThreads, 0, st>>>(rewards, values, dones, next_value, next_done, weights, T, E, D, envs_per_cta, (float)gamma,
                                                      (float)(gamma * gae_lambda), use_gae ? 1 : 0, returns, advantages);
    return check_launch("morl_vector_gae_f32");
}

extern "C" int morl_vector_gae_objectives_f32(const float* rewards, const float* values, const float* dones, const float* next_value,
                                              const float* next_done, int T, int E, int D, double gamma, double gae_lambda, float* returns,
                                              float* advantages, void* stream) {
    using namespace morl;
    MORL_REQUIRE(rewards && values && dones && next_value && next_done && returns && advantages, MORL_ERR_NULL,
                 "morl_vector_gae_objectives_f32: NULL pointer argument");
    MORL_REQUIRE(T > 0 && E > 0 && D > 0, MORL_ERR_SHAPE, "morl_vector_gae_objectives_f32: bad shape T=%d E=%d D=%d", T, E, D);
    MORL_REQUIRE(D <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "morl_vector_gae_objectives_f32: D=%d > %d", D, MORL_MAX_D);
    const int envs_per_cta = kGaeLanes / D;
    const int blocks = (E + envs_per_cta - 1) / envs_per_cta;
    vector_gae_kernel<false><<<blocks, kGaeThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        rewards, values, dones, next_value, next_done, nullptr, T, E, D, envs_per_cta, (float)gamma, (float)(gamma * gae_lambda), 1, returns,
        advantages);
    return check_launch("morl_vector_gae_objectives_f32");
}

extern "C" int morl_ppo_loss_f32(const float* mean, const float* logstd, const float* value, const float* actions, const float* old_logprob,
                                 const float* advantages, const float* returns, const float* old_values, int M, int A, int D, float clip_coef,
                                 float ent_coef, float vf_coef, int norm_adv, int clip_vloss, float* loss_out, float* dmean, float* dlogstd,
                                 float* dvalue, float* stats, void* stream) {
    using namespace morl;
    MORL_REQUIRE(mean && logstd && value && actions && old_logprob && advantages && returns && loss_out && dmean && dlogstd && dvalue && stats,
                 MORL_ERR_NULL, "morl_ppo_loss_f32: NULL pointer argument");
    MORL_REQUIRE(!clip_vloss || old_values, MORL_ERR_NULL, "morl_ppo_loss_f32: clip_vloss needs old_values");
    MORL_REQUIRE(M > 0 && A > 0 && D > 0, MORL_ERR_SHAPE, "morl_ppo_loss_f32: bad shape M=%d A=%d D=%d", M, A, D);
    MORL_REQUIRE(!norm_adv || M >= 2, MORL_ERR_SHAPE, "morl_ppo_loss_f32: advantage normalisation needs M >= 2 rows (unbiased std), got M=%d", M);
    MORL_REQUIRE(A <= kPpoMaxA, MORL_ERR_UNSUPPORTED, "morl_ppo_loss_f32: A=%d > %d", A, kPpoMaxA);
    MORL_REQUIRE(D <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "morl_ppo_loss_f32: D=%d > %d", D, MORL_MAX_D);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ppo_loss_kernel<<<1, kPpoThreads, 0, st>>>(mean, logstd, value, actions, old_logprob, advantages, returns, old_values, M, A, D, clip_coef, ent_coef,
                                               vf_coef, norm_adv ? 1 : 0, clip_vloss ? 1 : 0, loss_out, dmean, dlogstd, dvalue, stats);
    return check_launch("morl_ppo_loss_f32");
}
