/*
 * morl_b200.h -- C-ABI of libmorl_b200.so: the H100 (sm_90a) update engine for the batched
 * multi-objective value-update hot path of LucasAlegre/morl-baselines (reference @ a8acdbb).
 *
 * The reference has NO plugin / FFI layer (SURVEY.md section 8(b)): its boundary is the Python class API.
 * Each entry point below therefore replaces an *inline tensor-op sequence* of the reference; the
 * file:line it replaces is cited per function (paths relative to the reference root).
 *
 * Conventions (all entry points):
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch); the library never allocates,
 *     frees or retains device memory; tensors are contiguous row-major, base pointers 16-byte aligned;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it; no host sync, no
 *     allocation => safe under CUDA-graph capture; re-entrant (no mutable global state);
 *   - return value: 0 = success; negative = MORL_ERR_* argument error; positive = cudaError_t of
 *     the launch.  morl_last_error() returns a thread-local message for the last non-zero return;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point returns an error.
 *
 * Row-index maps.  Several per-row inputs of the reference are broadcast by `Tensor.repeat` (tile) or
 * `repeat_interleave` (block).  Instead of materialising them, an input X with x_rows < N rows is
 * addressed as
 *      MORL_MAP_TILE  : X[k % x_rows]            (reference: b_rewards.repeat(num_sample_w, 1), envelope.py:285-291)
 *      MORL_MAP_BLOCK : X[k / (N / x_rows)]      (reference: sampled_w.repeat_interleave(B, 0), envelope.py:284)
 *   x_rows == N is the identity under both maps.
 *
 * Scalarisation arithmetic (`dot_mode`).  s = w . q over D objectives, fp32:
 *      MORL_DOT_UNFUSED : ((w0*q0 + w1*q1) + w2*q2) + ...   every op rounded (IEEE, no contraction).  This is
 *                         bit-equal to the reference's th.einsum on CPU for small products (N_cols < 128),
 *                         e.g. the reference default num_sample_w=4 and every max_action / gpi_action call.
 *      MORL_DOT_PAIRFMA : fl(fma(w1,q1, fl(w0*q0)) + fl(w2*q2))   (D==3 only) -- bit-equal to what MKL's sgemm
 *                         produces for th.einsum("br,bwar->bwa") on the build container's AVX-512 CPU once
 *                         W*A >= 192 (probe in DESIGN.md); offered so golden vectors of the real reference at the
 *                         north-star shape can be matched bit-for-bit.
 *      MORL_DOT_FMA     : fma(w2,q2, fma(w1,q1, fl(w0*q0)))   the GPU-native chain (what cuBLAS would do).
 *   argmax / argmin are always FIRST-occurrence (th.max / th.argmax / th.argmin semantics).
 *
 * Selection rules of the four per-row targets below (greedy_td, critic_min_td, gpi_envelope, actor_critic_td):
 *   - ties: the argmax over candidates keeps the lowest index among equal scores (for gpi_envelope the joint index
 *     p*A + a, also when the tied candidates are walked by different lanes); the argmin over nets keeps the lowest net;
 *   - NaN: the argmax starts from -inf and only a strictly greater score replaces it, so a NaN score never wins.  The
 *     argmin over nets starts from net 0's score: a NaN at a later net never replaces it, a NaN at net 0 stays and then
 *     loses the argmax.  (th.argmax / th.argmin would return the NaN; the two differ only once values have diverged.)
 *     MORL_AC_ELEMENTWISE_MIN and MORL_AC_SCALAR_MIN take fminf, which ignores a NaN operand;
 *   - -inf: a row whose every score is -inf or NaN takes candidate 0 (action 0; for critic_min_td / gpi_envelope with
 *     the critic-min net of that candidate), as th.argmax does for an all -inf row;
 *   - w_map / r_map address w [w_rows, D] and reward / done [r_rows] by the row-index maps above: TILE row k % rows,
 *     BLOCK row k / (N / rows) (N = B for gpi_envelope); rows must divide N, and rows == N or rows == 1 mean the same
 *     under both maps.
 */
#ifndef MORL_B200_H_
#define MORL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MORL_B200_VERSION 200 /* 0.2.0 */

#if defined(__GNUC__)
#define MORL_API __attribute__((visibility("default")))
#else
#define MORL_API
#endif

/* argument errors (negative); positive returns are cudaError_t values */
#define MORL_OK 0
#define MORL_ERR_NULL (-1)        /* required pointer is NULL */
#define MORL_ERR_SHAPE (-2)       /* non-positive / inconsistent dimension */
#define MORL_ERR_ALIGN (-3)       /* base pointer not 16-byte aligned */
#define MORL_ERR_UNSUPPORTED (-4) /* dimension outside the compiled range (D > 8, A > 64, ...) */
#define MORL_ERR_NO_DEVICE (-5)   /* no CUDA device / wrong architecture */

#define MORL_DOT_UNFUSED 0
#define MORL_DOT_FMA 1
#define MORL_DOT_PAIRFMA 2

#define MORL_MAP_TILE 0
#define MORL_MAP_BLOCK 1

#define MORL_ROWS_REFERENCE 0 /* effective-batch row k = i*B + b  (reference order, envelope.py:284-291) */
#define MORL_ROWS_BMAJOR 1    /* effective-batch row k = b*W + i  (coalesced order used by the fused update)  */

#define MORL_MAX_D 8
#define MORL_MAX_A 64

MORL_API int morl_version(void);
MORL_API const char* morl_last_error(void);
/* number of SMs of the current device (132 on H100 SXM), or a negative MORL_ERR_* */
MORL_API int morl_device_sm_count(void);

/* ------------------------------------------------------------------------------------------------
 * Fused envelope-max TD target.   Replaces Envelope.envelope_target (multi_policy/envelope/envelope.py:404-440)
 * + the vector Bellman line (envelope.py:298), evaluated on the B*W DISTINCT (s'_b, w_j) rows instead of the
 * reference's B*W^2 tiled rows (SURVEY.md headline 2).
 *   q_online, q_target : f32 [B, W, A, D]   Q(s'_b, w_j)[a, :] of the online / target net (row b*W + j)
 *   wset               : f32 [W, D]         sampled weight vectors
 *   reward             : f32 [B, D], done : f32 [B]
 * For every (i, b):  (j*, a*) = first argmax_{j,a} wset[i] . q_online[b, j, a, :]
 *                    target[k, :] = reward[b, :] + ((1 - done[b]) * gamma) * q_target[b, j*, a*, :]   (unfused)
 * with k = i*B + b (MORL_ROWS_REFERENCE) or b*W + i (MORL_ROWS_BMAJOR).
 *   target_out : f32 [W*B, D];  pref_out, act_out : int32 [W*B] or NULL  (reference keeps them as int64, :424-426)
 */
MORL_API int morl_envelope_td_f32(const float* q_online, const float* q_target, const float* wset, const float* reward,
                         const float* done, float gamma, int B, int W, int A, int D, int dot_mode, int row_order,
                         float* target_out, int32_t* pref_out, int32_t* act_out, void* stream);

/* Double-DQN target with a per-row weight.  Replaces Envelope.ddqn_target (envelope.py:442-463) + :298, and the
 * non-GPI branch of GPIPD._reset_priorities (multi_policy/gpi_pd/gpi_pd.py:648-656).
 *   q_select, q_eval : f32 [N, A, D];  w : f32 [w_rows, D];  reward : f32 [r_rows, D] or NULL;  done : f32 [r_rows]
 *   a* = first argmax_a w_k . q_select[k, a, :];   out[k] = q_eval[k, a*, :]  (then Bellman if reward != NULL)
 */
MORL_API int morl_greedy_td_f32(const float* q_select, const float* q_eval, const float* w, int w_rows, int w_map,
                       const float* reward, const float* done, int r_rows, int r_map, float gamma, int N, int A,
                       int D, int dot_mode, float* target_out, int32_t* act_out, void* stream);

/* GPI-PD / GPI-LS critic-min target.  Replaces GPIPD.update's target block (gpi_pd.py:445-463):
 *   q_nets : f32 [n_nets, N, A, D] target nets;  n*(k,a) = first argmin_n w_k . q_nets[n,k,a,:];
 *   Q~[k,a,:] = q_nets[n*,k,a,:];  a* = first argmax_a w_k . Q~[k,a,:];  out = reward + ((1-done)*gamma) * Q~[k,a*,:]
 */
MORL_API int morl_critic_min_td_f32(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map,
                           const float* reward, const float* done, int r_rows, int r_map, float gamma, int N,
                           int A, int D, int dot_mode, float* target_out, int32_t* act_out, void* stream);

/* GPI envelope over a policy/weight-support set with per-row weights.  Replaces GPIPD._envelope_target
 * (gpi_pd.py:662-690), GPIPD.gpi_action (gpi_pd.py:564-582; n_nets = 1, reward = NULL), its batched twin in
 * _rollout_dynamics (gpi_pd.py:379-387) and the M x M GPI evaluation of GPIPDContinuousAction.eval
 * (multi_policy/gpi_pd/gpi_pd_continuous_action.py:464-478).
 *   q_nets : f32 [n_nets, B, P, A, D];  w : f32 [w_rows, D]
 *   per (b,p,a): critic-min over n as above (scalarised with w_b), then (p*, a*) = first joint argmax_{p,a}
 *   out[b,:] = Q~[b,p*,a*,:]  (Bellman applied iff reward != NULL);  policy_out / act_out : int32 [B] or NULL
 */
MORL_API int morl_gpi_envelope_f32(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map,
                          const float* reward, const float* done, int r_rows, int r_map, float gamma, int B, int P,
                          int A, int D, int dot_mode, float* out, int32_t* policy_out, int32_t* act_out,
                          void* stream);

/* Actor-critic vector targets (continuous-action algorithms), three "min over critics" rules (SURVEY App. A.4):
 *   MORL_AC_ELEMENTWISE_MIN : CAPQL  (multi_policy/capql/capql.py:326-331)  min_n per objective, - alpha*logp, vector target
 *   MORL_AC_SCALAR_MIN      : MOSAC  (single_policy/ser/mosac_continuous_action.py:435-442) scalarise, min, - alpha*logp;
 *                             out is [N] and the reward is scalarised with w as well
 *   MORL_AC_ARGMIN_GATHER   : GPI-PD continuous / TD3 (gpi_pd_continuous_action.py:397-403) first argmin_n w.q_n, gather vector
 *   q_nets : f32 [n_nets, N, D];  logp : f32 [N] or NULL;  w : [w_rows, D] (unused for ELEMENTWISE_MIN)
 */
#define MORL_AC_ELEMENTWISE_MIN 0
#define MORL_AC_SCALAR_MIN 1
#define MORL_AC_ARGMIN_GATHER 2
MORL_API int morl_actor_critic_td_f32(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map,
                             const float* reward, const float* done, const float* logp, float alpha, float gamma,
                             int N, int D, int variant, float* target_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused TD loss + gradient seed + PER priority for Envelope.  Replaces envelope.py:301-313 (gather taken action,
 * MSE, homotopy auxiliary loss) and :329-331 (|w . td| priorities of the first B rows, i.e. weight index 0).
 *   q_values : f32 [W*B, A, D] online net output on the effective batch (row order `row_order`)
 *   action   : int32 [B];  target_q : f32 [W*B, D];  wset : f32 [W, D]
 *   homotopy_lambda_dev : optional device f32 [1]; when non-NULL the kernels read lambda from it instead of the by-value argument, so a
 *              captured CUDA graph stays valid while the homotopy schedule (envelope.py:351-358) changes lambda every update
 *   loss_out : f32 [1] = (1-lambda)*mean((q-t)^2) + lambda*mean((w.q - w.t)^2)
 *   grad_q   : f32 [W*B, A, D] = d loss / d q_values (dense; zero off the taken action), or NULL
 *   q_taken  : f32 [W*B, D] the gathered Q(s,a) (optional, NULL to skip)
 *   prio_out : f32 [B] = | wset[0] . (q - t) | for rows with i == 0, or NULL
 *   workspace: device scratch of morl_td_workspace_bytes(W*B) bytes (no initialisation required)
 */
MORL_API size_t morl_td_workspace_bytes(int n_rows);
MORL_API int morl_td_mse_priority_f32(const float* q_values, const int32_t* action, const float* target_q,
                             const float* wset, float homotopy_lambda, const float* homotopy_lambda_dev, int B, int W, int A,
                             int D, int row_order, float* loss_out, float* grad_q, float* q_taken, float* prio_out, void* workspace,
                             void* stream);

/* Huber-style TD loss of GPI-PD.  Replaces gpi_pd.py:469-487 per net and :507-520 (priority = | w . max_n |delta_n| |).
 *   q_values : f32 [n_nets, N, A, D];  action : int32 [a_rows] (tile map);  target_q : f32 [N, D]
 *   target_q_gpi : f32 [N, D] or NULL (gpi_pd=True -> priorities from the GPI envelope target)
 *   loss_out : f32 [1] = (1/n_nets) * sum_n mean( where(|d|<mp, 0.5 d^2, mp |d|) )   (common/networks.py:90-100)
 *   grad_q   : f32 [n_nets, N, A, D] or NULL;   prio_out : f32 [p_rows] (first p_rows rows), raw |w . err| before clip/pow
 *   |d| == min_priority exactly takes the linear branch (mp |d|; the gradient is +-mp either way); d == +-0 adds nothing and
 *   has a zero gradient.  action row k is action[k % a_rows]; the priority weight of row k is w[TILE or BLOCK map of w_map].
 */
MORL_API int morl_td_huber_priority_f32(const float* q_values, int n_nets, const int32_t* action, int a_rows,
                               const float* target_q, const float* target_q_gpi, const float* w, int w_rows,
                               int w_map, float min_priority, int N, int A, int D, int p_rows, float* loss_out,
                               float* grad_q, float* prio_out, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Discrete-action MOSAC (single_policy/ser/mosac_discrete_action.py).  A fourth "min over critics" rule next to the three of
 * morl_actor_critic_td_f32: the soft value is an expectation under the actor's softmax over ALL actions, not a value at one
 * sampled action.  Shapes: q_nets f32 [n_nets, N, A, D]; logits f32 [N, A]; w [w_rows, D] under w_map; A <= 256, D <= 8 (larger
 * shapes return MORL_ERR_UNSUPPORTED).  alpha (and log_alpha) are DEVICE f32 [1], read at run time, so a captured CUDA graph stays
 * valid while the temperature is tuned.  Per row k, actions walked in ascending order:
 *   mx = max_a x[a] (NaN propagates);  s = sum_a e^(x[a] - mx);  logp[a] = (x[a] - mx) - log s;  p[a] = e^(x[a] - mx) / s
 *     (torch's max-subtracted log_softmax / softmax; e^ and log are the library's own portable fp32 routines, <= 2 ulp)
 *   m[a] = min_n (w . q_n[k, a, :])  scalarised in MORL_DOT_UNFUSED, the arithmetic morl_actor_critic_td_f32 uses for MOSAC's
 *     th.matmul; the min follows th.min and PROPAGATES NaN (unlike the fminf of MORL_AC_SCALAR_MIN, which ignores a NaN operand)
 *   -inf logit: p[a] = 0 and logp[a] = -inf; such an action is left out of every sum below and its gradient is 0 (the reference
 *     would compute 0 * -inf = NaN and poison the row).  A row whose max is +-inf or NaN is NaN throughout, as in torch.
 * morl_discrete_sac_target_f32 (:452-464):
 *   v = sum_a p[a] * (m[a] - alpha * logp[a]);  target_out[k] = w.r + ((1 - done) * gamma) * v     reward f32 [N, D], done f32 [N]
 * morl_discrete_sac_actor_loss_f32 (:478-498), q_nets the ONLINE critics at s evaluated after the critic step:
 *   f[a] = alpha * logp[a] - m[a];  l_k = sum_a p[a] f[a]
 *   actor_loss_out[0] = sum_k l_k / (N*A)          (the reference's .mean() of a [N, A] tensor)
 *   dlogits [N, A] (or NULL) = p[a] * (f[a] - l_k) / (N*A)   (closed form: softmax Jacobian with sum_a p = 1)
 *   log_alpha non-NULL (autotune): t = -e^log_alpha, u[a] = logp[a] + target_entropy,
 *     alpha_loss_out[0] = sum_k sum_a p[a] * (t * u[a]) / (N*A);  dlog_alpha_out[0] = t * sum_k sum_a p[a] u[a] / (N*A)
 *   Row sums are reduced deterministically: fixed 256-row block partials in float, then one final sum in double.
 *   workspace: device scratch of morl_discrete_sac_workspace_bytes(N) bytes (no initialisation required)
 */
MORL_API int morl_discrete_sac_target_f32(const float* q_nets, int n_nets, const float* logits, const float* w, int w_rows, int w_map,
                                          const float* reward, const float* done, const float* alpha, float gamma, int N, int A, int D,
                                          float* target_out, void* stream);
MORL_API size_t morl_discrete_sac_workspace_bytes(int n_rows);
MORL_API int morl_discrete_sac_actor_loss_f32(const float* logits, const float* q_nets, int n_nets, const float* w, int w_rows,
                                              int w_map, const float* alpha, const float* log_alpha, float target_entropy, int N,
                                              int A, int D, float* actor_loss_out, float* dlogits, float* alpha_loss_out,
                                              float* dlog_alpha_out, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Host halves of the replay path (CPU code in the same library; no CUDA call, usable without a device).
 *
 * Prioritised replay sum tree, reference common/prioritized_buffer.py:12-82 (class SumTree).  `tree` is ONE float64 array of
 * 2^n_levels - 1 nodes: level l (2^l nodes, l = 0 the root, l = n_levels - 1 the leaves) starts at element 2^l - 1.
 *   morl_host_sumtree_walk      : SumTree.sample after the uniform draw (:35-49): descend for each query value -> leaf index.
 *   morl_host_sumtree_batch_set : SumTree.batch_set (:73-82): np.unique(index, return_index) then node += (new - old) on every
 *                                 level in array order -- the same float64 operations in the same order, so the tree (and the
 *                                 indices later sampled from it) is bit-identical to the reference's.
 * Minibatch packing, reference common/buffer.py:84-94 (fancy-index gathers before the host->device copies):
 *   morl_host_gather_rows       : dst[i, :] = src[index[i], :] for rows of row_bytes bytes (dst: pinned staging memory).
 *   morl_host_gather_u8_to_i32  : same for uint8 action rows, widened to int32 (the reference's callers call .long()). */
MORL_API int morl_host_sumtree_walk(const double* tree, int n_levels, const double* queries, int n, long long* out_index);
MORL_API int morl_host_sumtree_batch_set(double* tree, int n_levels, const long long* index, const double* priority, int n);
MORL_API int morl_host_gather_rows(const void* src, long long row_bytes, const long long* index, int n, void* dst);
MORL_API int morl_host_gather_u8_to_i32(const unsigned char* src, long long row_elems, const long long* index, int n, int* dst);

/* ------------------------------------------------------------------------------------------------
 * Device-resident replay: index gather.  Replaces the 5 fancy-index gathers + 6 host->device copies of
 * ReplayBuffer.sample (common/buffer.py:82-94) / PrioritizedReplayBuffer.sample (common/prioritized_buffer.py:160-166).
 *   stores: obs/next_obs f32 [cap, obs_dim], action u8|f32 [cap, act_dim], reward f32 [cap, rew_dim], done f32 [cap]
 *   idx : int64 [B];  outputs are [B, *];  discrete actions (act_is_u8 != 0) are widened to int32.
 */
MORL_API int morl_replay_gather(const float* obs_store, const float* next_obs_store, const void* act_store,
                       const float* rew_store, const float* done_store, const int64_t* idx, int B, int obs_dim,
                       int act_dim, int rew_dim, int act_is_u8, int64_t capacity, float* obs_out,
                       float* next_obs_out, void* act_out, float* rew_out, float* done_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pareto non-dominated mask (maximisation).  Replaces get_non_pareto_dominated_inds (common/pareto.py:34-57):
 *   keep[i] = 1 iff no OTHER value weakly dominates pts[i] (only exact copies are >= in every coordinate) and,
 *   when remove_duplicates != 0, i is the first index holding its value.  Comparisons are exact in the input dtype;
 *   a row containing NaN is never kept.  pts : [N, D] row-major; keep : uint8 [N].  D <= MORL_MAX_D.
 */
MORL_API int morl_pareto_mask_f32(const float* pts, int N, int D, int remove_duplicates, uint8_t* keep, void* stream);
MORL_API int morl_pareto_mask_f64(const double* pts, int N, int D, int remove_duplicates, uint8_t* keep, void* stream);

/* Fixed-shape records for the ONE all-gather of per-rank non-dominated fronts per evaluation round (BASELINE.json north_star; the
 * reference has no multi-GPU path -- the call it replaces is the single-process archive update of multi_policy/morld/morld.py:306-335).
 *   record (float64) = [ count | cap x d rows | n_extra extras ]
 * morl_front_pack_f64   : rows of pts [n, d] with keep[i] != 0 (keep NULL = all), in input order; count is NOT clipped to cap (overflow is
 *                         visible to every rank after the gather); unused rows are -inf (dominated by any real point).  One block.
 * morl_front_unpack_f64 : gathered [world][1 + cap*d + n_extra] -> pts_out [world*cap, d] (input of the global prune) and
 *                         meta_out [world][1 + n_extra] (every rank's count and extras, contiguous).
 * No host synchronisation, no allocation: the whole exchange is stream-ordered. */
MORL_API int morl_front_pack_f64(const double* pts, const uint8_t* keep, int n, int d, int cap, const double* extras, int n_extra, double* rec,
                                 void* stream);
MORL_API int morl_front_unpack_f64(const double* gathered, int world, int d, int cap, int n_extra, double* pts_out, double* meta_out, void* stream);

/* Exact hypervolume (maximisation) of the points with keep[i] != 0 (keep NULL = all) above the reference point `ref` [d], 1 <= d <= 3,
 * n <= 2048, float64, one launch, result in *out (device): replaces `hypervolume(ref_point, points)` of the reference
 * (common/performance_indicators.py:15-25; pymoo's exact HV) for fronts that already live on the device.  Points that do not exceed
 * `ref` in every objective contribute nothing; dominated points are harmless (the volume is that of the union of boxes). */
MORL_API int morl_hypervolume_f64(const double* pts, const uint8_t* keep, int n, int d, const double* ref, double* out, void* stream);

/* Batched exact hypervolume (maximisation, float64) of "a base set plus one candidate" for every candidate, in one launch (one block per
 * candidate): IPRO's hypervolume improvements of its sampled lower points (multi_policy/ipro/ipro.py:212-226) and its other volumes.
 *   n_cand >= 1 : out[k] = volume of base [n_base, d] U { cand[k] } (cand [n_cand, d]) above ref [d], k < n_cand
 *   n_cand == 0 : out[0] = volume of base alone (cand may be NULL)
 * Points count as in morl_hypervolume_f64: q = p - ref clipped at 0; a point that does not exceed ref in every objective, or holds a NaN,
 * spans nothing.  d = 4 slices over the fourth objective, each slab a 3-D volume by the same sweep (O(n^3) per set); results do not depend
 * on the grid (fixed-shape reductions, no atomics), and with n_cand == 0 and d <= 3 they equal morl_hypervolume_f64's bit for bit.
 * Supported range (morl_hypervolume_batch_supported, no device needed: 1 if supported, else 0): 1 <= d <= 4 and 0 <= n_base <= 2048 for
 * d <= 3, <= 512 for d = 4; anything else returns MORL_ERR_UNSUPPORTED (compute on the host instead). */
MORL_API int morl_hypervolume_batch_supported(int n, int d);
MORL_API int morl_hypervolume_batch_f64(const double* base, int n_base, const double* cand, int n_cand, int d, const double* ref, double* out,
                                        void* stream);

/* Pareto Q-learning's set table (multi_policy/pareto_q_learning/pql.py), caller-owned device tensors for S states, A actions, set
 * capacity K and d objectives:  nd f64 [S, A, K, d] and nd_count int32 [S, A] (the stored set ND[s][a]: its first nd_count rows; start
 * with count 1 and the zero vector), avg_reward f64 [S, A, d], counts f64 [S, A], status int32 [3] (zeroed by the caller).
 * Q-set(s, a) = { avg_reward[s, a] + gamma * v : v in ND[s][a] }, each coordinate rounded as numpy does (gamma * v, then the add).
 * morl_pql_update_f64 : one reference step (pql.py:260-262), one CTA:  counts[s, a] += 1;  ND[s][a] = ND(U_a' Q-set(s_next, a'));
 *   avg_reward[s, a] += (reward - avg_reward[s, a]) / counts[s, a] (subtract, divide, add: one IEEE operation each).  ND keeps a point
 *   iff no distinct point is >= it in every coordinate, and one copy of equal points (within and across actions).  The set is stored in
 *   canonical order: descending coordinate sum (added left to right), ties lexicographically descending, so equal sets are equal bytes.
 *   The union is staged on chip before anything is written, so s_next == s is safe.  If more than K points survive, nothing is written
 *   but status: { needed size, s, a } when status[0] was 0 (the first overflow is kept).  reward: HOST pointer to d doubles, passed to
 *   the kernel by value (no copy to the device).  s, s_next in [0, S), a in [0, A), else MORL_ERR_SHAPE.
 * morl_pql_score_f64 : scores f64 [A] of `state`, one CTA per action.
 *   mode MORL_PQL_HYPERVOLUME (pql.py:143-154): scores[a] = exact volume of Q-set(state, a) above ref (HOST pointer to d doubles, passed
 *     by value), counted as morl_hypervolume_batch_f64 counts it: a point that does not exceed ref in every objective spans nothing.  Equal
 *     sets give bit-identical volumes.
 *   mode MORL_PQL_CARDINALITY (pql.py:122-141): scores[a] = number of points of ND(U_a' Q-set(state, a')) equal to a point of
 *     Q-set(state, a) (a point shared by several actions counts for each); ref may be NULL.
 *   Integer counts and fixed-shape reductions: no atomics, results do not depend on the grid.
 * Supported range (morl_pql_supported, no device needed: 1 if supported, else 0): 1 <= A <= 16, 1 <= K <= 256, A * K <= 2048 and
 *   1 <= d <= MORL_MAX_D, with d <= 4 for MORL_PQL_HYPERVOLUME; the update needs the MORL_PQL_CARDINALITY range.  Anything else returns
 *   MORL_ERR_UNSUPPORTED. */
#define MORL_PQL_HYPERVOLUME 0
#define MORL_PQL_CARDINALITY 1
MORL_API int morl_pql_supported(int n_actions, int cap, int d, int mode);
MORL_API int morl_pql_update_f64(double* nd, int* nd_count, double* avg_reward, double* counts, int* status, int S, int A, int K, int d, int s,
                                 int a, int s_next, double gamma, const double* reward, void* stream);
MORL_API int morl_pql_score_f64(const double* nd, const int* nd_count, const double* avg_reward, int S, int A, int K, int d, int state,
                                double gamma, int mode, const double* ref, double* scores, void* stream);

/* Multi-policy scalarised Q-learning (multi_policy/multi_policy_moqlearning/mp_mo_q_learning.py with single_policy/ser/mo_q_learning.py and
 * common/model_based/tabular_model.py), caller-owned device tensors for S states, P policy slots, A actions, d objectives, M model pairs and
 * K outcomes per pair:  q f64 [S, P, A, d] (zero where a policy never visited a state), visited u8 [S, P], pairs int32 [M, 3] (state,
 * action, number of outcomes; zeroed), outcomes int32 [M, K, 2] (next state, terminal), counts int64 [M, K] (zeroed), out_reward
 * f64 [M, K, d], tree f64 [2^18 - 1] (the reference's SumTree(max_size=1e5), zeroed), status int32 [2] (zeroed).  w . v adds the products
 * left to right, one IEEE operation each; every update is numpy's expression order with no FMA contraction.
 * morl_moq_act_f64 : n rows (HOST arrays, passed by value: no copy to the device), one block per row.  policy[i] >= 0: argmax over actions
 *   of w . q[state, policy]; policy[i] == -1: GPI, argmax over the stacked [n_policies, A] values in row-major order.  First maximum wins
 *   (numpy's argmax, a NaN first); a state the policy never visited, and state -1, scores 0.  out int32 [n, 2] = (action, visited) where
 *   visited is 1 iff an own-policy row's state is in the policy's table; value f64 [n] (may be NULL) = the winning value.
 * morl_moq_step_f64 : one environment step of policy p (mo_q_learning.py:173-208) in one block: visit s and s_next, greedy action at
 *   s_next (GPI over the first n_policies with MORL_MOQ_GPI), td = r + ((1 - terminal) * gamma) * q[s_next, p, a'] - q[s, p, a],
 *   q[s, p, a] += lr * td.  With MORL_MOQ_MODEL the transition enters the model as outcome `outcome` of pair `pair` (the caller keys both;
 *   pair < n_pairs), then n_updates Dyna updates follow, each on a pair drawn uniformly (pick[j], HOST) or, with MORL_MOQ_PRIORITIZE, by
 *   the tree walk of query root * u[j] (HOST), an outcome drawn as random.choices does with random() = choice[j] (HOST), and the same TD
 *   update.  With MORL_MOQ_PRIORITIZE every update also sets the pair's leaf to max(|r.w + ((1 - terminal) gamma) max_scalar_q(s', w)
 *   - q[s, p, a].w|, min_priority) ** alpha.  w and reward: HOST pointers to d doubles, passed by value.  A walk that lands on a leaf
 *   >= n_pairs (the reference's IndexError) writes status = {1, leaf} and stops; while status[0] != 0 the call changes nothing.  More than
 *   64 Dyna updates run as consecutive launches.
 * Supported range (morl_moq_supported, no device needed): 1 <= A <= 64, 1 <= d <= MORL_MAX_D; else MORL_ERR_UNSUPPORTED. */
#define MORL_MOQ_GPI 1
#define MORL_MOQ_MODEL 2
#define MORL_MOQ_PRIORITIZE 4
MORL_API int morl_moq_supported(int n_actions, int d);
MORL_API int morl_moq_act_f64(const double* q, const unsigned char* visited, int S, int P, int A, int d, int n_policies, const int* state,
                              const int* policy, const double* w, int n, int* out, double* value, void* stream);
MORL_API int morl_moq_step_f64(double* q, unsigned char* visited, int* pairs, int* outcomes, long long* counts, double* out_reward, double* tree,
                               int* status, int S, int P, int A, int d, int M, int K, int n_policies, int p, int s, int a, int s_next, int terminal,
                               int pair, int outcome, int n_pairs, const double* w, const double* reward, int flags, double gamma, double lr,
                               double min_priority, double alpha, int n_updates, const int* pick, const double* u, const double* choice,
                               void* stream);

/* Corner weights of a convex coverage set (OLS / GPI-LS weight selection).  Replaces compute_corner_weights
 * (multi_policy/linear_support/linear_support.py:295-349), which enumerates with cdd the vertices of
 *   { (w, u) : V w <= u 1,  w >= 0,  sum w = 1 }.
 * Exact enumeration over the C(n+d, d) d-subsets of the n + d inequality rows, one d x d float64 solve each; a degenerate vertex is
 * emitted once (by its lexicographically first basis).  V : f64 [n, d] row-major (the caller rounds it, np.round(., 4));
 * verts : f64 [cap, d+1], (w, u) per vertex in no particular order (may be NULL iff cap == 0); count : device int [1] = number of
 * vertices found, NOT clipped to cap (grow the buffer and launch again).  2 <= d <= MORL_MAX_D, n >= 1, and
 * C(n+d, d) <= MORL_CORNER_MAX_CANDIDATES (2^31: e.g. d 6 with n <= 94, d 8 with n <= 58), else MORL_ERR_UNSUPPORTED. */
#define MORL_CORNER_MAX_CANDIDATES 2147483648ULL
MORL_API int morl_corner_weights_f64(const double* V, int n, int d, double* verts, int cap, int* count, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Multi-tensor target-network sync.  Replaces polyak_update (common/networks.py:121-139):
 *   tau == 1 : target <- param;  else target <- fma(tau, param, fl((1 - tau) * target))   (mul_ then ATen's fused add(alpha))
 *   params / targets : device arrays of n_tensors device pointers; sizes : device int64 [n_tensors]
 */
MORL_API int morl_polyak_f32(const float* const* params, float* const* targets, const int64_t* sizes, int n_tensors,
                    int64_t max_size, double tau, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Device-resident prioritised-replay sum tree (SURVEY.md 8(f)1), bit-identical to the reference's numpy tree (common/prioritized_buffer.py:
 * 12-82): float64, level l (2^l nodes) at element 2^l - 1 of `tree`, root first -- the layout of morl_host_sumtree_*.
 *   morl_sumtree_walk_f64       : SumTree.sample without the RNG (:40-54): query_i = scale_by_root ? tree[0] * u[i] : u[i]  (the host draws
 *                                 u with np.random.random_sample, the same stream np.random.uniform(0, root) consumes), level walk with
 *                                 strict '>' going right; out_index int64 [n].
 *   morl_sumtree_batch_set_f64  : SumTree.batch_set (:66-82): np.unique first-occurrence semantics, diff = new - leaf, then the per-level
 *                                 additions of np.add.at in sorted-leaf order; n <= 2048 indices per call.  *err_flag (device int) is set
 *                                 to 1 if an index is out of range.
 *   morl_sumtree_set_f64        : SumTree.set (:56-64; replay_buffer.add): one leaf, scalar arguments; use_min_priority != 0 takes the new
 *                                 priority from the buffer's current min_priority (device float64: the reference's python float until the first ratchet) instead
 *                                 of `priority`.
 *   morl_per_priority_f32       : p = fl32(fl32(raw + fl32(min_p)) ** alpha) (envelope.py:333; gpi_pd.py:523-525 callers pass their own raw),
 *                                 prio64 = (double) p for the tree, optional float32 copy, then *min_priority = max(*min_priority, max p)
 *                                 (prioritized_buffer.py:194).
 * All of them are single stream-ordered launches without host synchronisation: sample -> gather -> update -> priorities -> tree is one CUDA graph. */
MORL_API int morl_sumtree_walk_f64(const double* tree, int n_levels, const double* u, int n, int scale_by_root, long long* out_index, void* stream);
MORL_API int morl_sumtree_batch_set_f64(double* tree, int n_levels, const long long* index, const double* priority, int n, int* err_flag,
                                        void* stream);
MORL_API int morl_sumtree_set_f64(double* tree, int n_levels, long long index, double priority, int use_min_priority, const double* min_priority,
                                  int* err_flag, void* stream);
MORL_API int morl_per_priority_f32(const float* raw, int n, float alpha, double* min_priority, double* prio64, float* prio32, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FP32-accurate dense layers on the Hopper tensor cores (wgmma).  Replace the fp32 GEMMs behind the reference's nn.Linear layers
 * (common/networks.py:10-48; called from envelope.py:59-77 / :300, :420, :429 on the 65,536-row effective batch).
 * Every fp32 operand is carried as P 16-bit planes [P][rows][ld] (`plane_stride` elements between planes) whose sum reproduces it;
 * a product is the sum of the significant plane-by-plane MMAs with fp32 accumulation in registers (csrc/gemm_planes.cu):
 *   MORL_FMT_F16X2  : P = 2 fp16 planes of  scale * x  (scale: a power of two held in a DEVICE float, NULL = 1), 3 MMAs, exact to
 *                     2^-22; |scale * x| must stay below 65,504 -- beyond it the planes hold Inf/NaN (propagating to every output)
 *                     and morl_plane_overflow_count() becomes non-zero.  4 bytes / element.
 *   MORL_FMT_BF16X3 : P = 3 bf16 planes of x (fp32 exponent range, scale pointers normally NULL), 6 MMAs, exact to 2^-24.  6 bytes / element.
 * All scale arguments are device pointers so that a captured CUDA graph stays valid when the scales change.
 *
 * morl_amax_scale_f32 : *scale_out = 2^(target_exp - e) with max|src| < 2^e, i.e. scale * max|src| in [2^(target_exp-1), 2^target_exp)
 *                     (1 if src is all zero).  workspace: 8 bytes, ZERO before the first call (left zero again).
 * morl_split_planes : fp32 [rows, cols] (row stride ld_src; transposed read if `transpose`) -> planes [P][rows_pad][ldp] of scale * x,
 *                     zero padded.
 * morl_split_planes_multi : up to MORL_SPLIT_MAX_JOBS independent splits (all weight matrices of a network, plain and transposed) in
 *                     one launch; a job with auto_scale != 0 derives its scale from the largest magnitude of its own matrix
 *                     (scale * amax in [2^(target_exp-1), 2^target_exp)) and stores it in *scale.
 * morl_gemm_planes_f32 : C = act(A . B^T + bias),  A planes [P][M][K] (K-major), B planes [P][N_pad][K] (K-major weights);
 *                     K % 64 == 0 (f16x2) / K % 32 == 0 (bf16x3), N_pad % 32 == 0, N_pad <= 512 (wider than 256: two column units
 *                     [0, 256) and [256, N_pad) of a row tile, each bit-identical to a launch over that half).  The accumulator is multiplied by
 *                     1 / (a_scale * b_scale) before the bias.  Outputs: c_f32 [M, ldc] and/or c_planes [P][M][ldp] holding
 *                     c_scale * C (the operand format of the next layer).  relu != 0 applies max(x, 0).
 *                     ReLU bit masks (the only form of the ReLU-backward mask):
 *                     relu_bits_out [M][8] uint32 (N_pad <= 256) receives bit j of word (c & 1) * 4 + (c >> 1) = (C[m, 32 c + j] > 0) -- 32
 *                     bytes per row instead of the 512-byte activation row, words ordered so that the four chunks one epilogue thread
 *                     owns are one 16-byte load.  N_pad > 256: [M][16] words (the row pitch follows N_pad, not N: every 32-column
 *                     chunk below N_pad has a word, padding chunks included), bit j of word 8 * (c >> 3) + (c & 1) * 4 + ((c >> 1) & 3):
 *                     each 256-column half of the row keeps the 8-word order above, the second half's words after the first's.
 *                     relu_bits_in (same layout, written by the forward call of the layer or by
 *                     morl_pairs_relu_split_planes) zeroes the outputs whose bit is clear, i.e. relu'(x) = [x > 0] exactly as
 *                     torch's ReLU backward (reference networks.py:10-48 under autograd).  Both nullable, 16-byte aligned.
 *                     reverse_tiles != 0 walks the 128-row tiles from the last to the first: alternate it between the layers of
 *                     a chain so that a layer starts on the rows its producer wrote last (still in the 50 MB L2).
 *                     split_accumulators != 0: the leading products A0.B0 and the correction products accumulate in separate register
 *                     accumulators and are added once, correctly rounded, in the epilogue, so that only K/16 accumulations happen at
 *                     full magnitude; the price is that an output wider than 128 columns is computed as two column units (the
 *                     A tile is staged twice).
 */
#define MORL_FMT_BF16X3 0
#define MORL_FMT_F16X2 1
#define MORL_SPLIT_MAX_JOBS 16
typedef struct MorlSplitJob {
    const float* src;       /* fp32 [rows, cols], row stride ld_src */
    void* dst_planes;       /* 16-bit [P][rows_pad][ldp] */
    long long plane_stride; /* elements between planes */
    float* scale;           /* device float: read (auto_scale == 0; NULL = 1) or written first, then used (auto_scale != 0; must not be NULL) */
    int rows, cols, ld_src, transpose, rows_pad, ldp;
    int auto_scale, target_exp;
} MorlSplitJob;
MORL_API int morl_plane_overflow_count(int reset); /* >= 0: f16x2 range violations seen since the last reset (synchronises the device) */
MORL_API int morl_amax_scale_f32(const float* src, long long n, int target_exp, float* scale_out, void* workspace, void* stream);
MORL_API int morl_split_planes_multi(int fmt, const MorlSplitJob* jobs, int n_jobs, void* stream);
MORL_API int morl_split_planes(int fmt, const float* src, int rows, int cols, int ld_src, int transpose, void* dst_planes, int rows_pad,
                               int ldp, long long plane_stride, const float* scale, void* stream);
MORL_API int morl_gemm_planes_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                                  long long b_plane_stride, const float* b_scale, int M, int N, int N_pad, int K, const float* bias,
                                  int relu, float* c_f32, int ldc, void* c_planes, int ldp, long long c_plane_stride, const float* c_scale,
                                  int reverse_tiles, int split_accumulators, const void* relu_bits_in, void* relu_bits_out, void* stream);
/* Hidden layer Linear -> Dropout(p) -> LayerNorm -> ReLU of GPI-PD's Q-network (reference gpi_pd.py:41-76, networks.py:10-48) as ONE
 * K-major GEMM whose epilogue computes, per output row,  y = relu(LN(dropout(A . B^T / (a_scale b_scale) + bias)))  (csrc/gemm_planes.cu,
 * gemm_planes_kernel<FMT, 0, kEpiLn>).  Operands, scales, reverse_tiles, c_f32 / c_planes as in morl_gemm_planes_f32 with N_pad = N; the
 * re-split planes hold c_scale * y (c_scale applied after the ReLU: LayerNorm is not scale-invariant through eps).  N % 32 == 0, N <= 256.
 *   layer_norm != 0: two-pass fp32 mean and biased variance over the N columns of the row, (x - mean) rsqrt(var + ln_eps) gamma + beta;
 *                    ln_gamma / ln_beta [N] device vectors (NULL = 1 / 0).
 *   dropout (drop_seed != NULL): keep element (row, col) iff its Philox4x32-10 draw is >= round(drop_p 2^32), kept values times
 *                    float(1 / (1 - drop_p)); key = *drop_seed, counter = (*drop_offset, drop_salt, row, column group).  Seed and offset are
 *                    device-resident: advance the offset with morl_philox_advance inside the same stream (or captured graph) for fresh masks.
 *   drop_bits_out (nullable, 16-byte aligned): the keep mask as bits in the ReLU-bit layout ([M][8] uint32; bit set = kept).
 * With layer_norm = 0 and no dropout the outputs equal morl_gemm_planes_f32(relu = 1, split_accumulators = 0) bit for bit. */
MORL_API int morl_gemm_planes_ln_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* b_planes,
                                     long long b_plane_stride, const float* b_scale, int M, int N, int K, const float* bias, int layer_norm,
                                     const float* ln_gamma, const float* ln_beta, float ln_eps, float drop_p, const unsigned long long* drop_seed,
                                     const unsigned int* drop_offset, unsigned int drop_salt, float* c_f32, int ldc, void* c_planes, int ldp,
                                     long long c_plane_stride, const float* c_scale, int reverse_tiles, void* drop_bits_out, void* stream);
/* *offset += inc as one stream-ordered launch (the dropout pass counter of morl_gemm_planes_ln_f32; capture-safe). */
MORL_API int morl_philox_advance(unsigned int* offset, unsigned int inc, void* stream);
/* Several 256-wide hidden layers (Linear + ReLU) of one or two networks in ONE persistent launch (csrc/gemm_planes.cu: gemm_chain_kernel):
 * job (c, l):  act[c][l+1] = f(act[c][l] . W[c][l]^T + bias[c][l]),  planes in / planes out at the scale `act_scale`; f = ReLU (relu != 0:
 * forward chains, optionally recording the ReLU bit masks) or the ReLU-backward mask relu_bits_in[job] (dX chains of the backward pass:
 * G_{l-1} = (G_l . W_l) * relu'(H_{l-1}), biases NULL) --
 * bit-identical to n_chains * n_layers calls of morl_gemm_planes_f32 (c_scale = a_scale) -- but a CTA takes each of its 128-row tiles
 * through all layers, so every intermediate activation is re-read from the L2 it was just written to instead of from HBM, and the launch
 * prologue / drain is paid once.  Replaces the per-layer launches behind the reference's hidden nn.Linear + ReLU stack (networks.py:10-48) in the
 * no-grad passes (both networks at once: n_chains = 2) and in the training pass (n_chains = 1, with ReLU bit masks).
 *   act_planes [n_chains * (n_layers + 1)] : plane tensors [P][M][256] (host array of device pointers; index c * (n_layers + 1) + l);
 *   w_planes / w_scales / biases / relu_bits_in / relu_bits_out [n_chains * n_layers] (index c * n_layers + l; all but w_planes nullable, also per entry).
 *   k_first (0 = K): reduction length of layer 0 -- its input act[c][0] may be a NARROWER dense tensor [P][M][k_first] with weights [P][256][k_first]
 *   (plane strides M * k_first and 256 * k_first): the dX product of the 24-wide output layer as the first job of the backward chain.
 * morl_gemm_chain_supported: K == 256 (square 256-wide layers), M >= 256. */
MORL_API int morl_gemm_chain_supported(int fmt, int M, int K);
MORL_API int morl_gemm_chain_f32(int fmt, int n_chains, int n_layers, const void* const* act_planes, long long act_plane_stride, const float* act_scale,
                                 const void* const* w_planes, long long w_plane_stride, const float* const* w_scales, const float* const* biases,
                                 int relu, const void* const* relu_bits_in, void* const* relu_bits_out, int M, int K, int k_first, void* stream);
/* f16x2 chains run with the activation tile resident in shared memory (k_first then needs only be a multiple of 32); bf16x3 chains as above.
 * morl_gemm_chain_pairs_f32: the same forward chains (ReLU, f16x2), started from the separable first layer: the input of chain c is
 * relu(u[c][b] + v[c][j]) * act_scale for row b * W + j (u[c] [B][256], v[c] [W][256] fp32, 16-byte aligned) -- the planes
 * morl_pairs_relu_split_planes would write, built on chip instead.  acts[c * n_layers + l] ([P][B W][256]) receives the output of layer l
 * of chain c only when bit c * n_layers + l of store_mask is set (may be NULL otherwise); the others never leave shared memory. */
MORL_API int morl_gemm_chain_pairs_f32(int n_chains, int n_layers, const float* const* u, const float* const* v, int B, int W, const void* const* acts,
                                       long long act_plane_stride, const float* act_scale, const void* const* w_planes, long long w_plane_stride,
                                       const float* const* w_scales, const float* const* biases, void* const* relu_bits_out, unsigned int store_mask,
                                       void* stream);
/* Diagnostics (not part of the reference surface): per-role cycle counters of morl_gemm_planes_f32, summed over CTAs and launches
 * since the last reset; collected only when the environment variable MORL_GEMM_STATS=1 is set before the first GEMM call.
 * out8: [0] MMA thread waiting for TMA data, [1] waiting for the epilogue to free an accumulator, [2] MMA loop total,
 * [3] TMA thread waiting for a free stage, [4] epilogue waiting for an accumulator, [5] epilogue busy; [6], [7] reserved. */
MORL_API int morl_debug_gemm_stats(unsigned long long* out8, int reset);
/* GPI-PD Dyna planning (SURVEY 8(f)3): everything between the last layer of the probabilistic ensemble and the imagined transition in ONE
 * pass (reference common/model_based/probabilistic_ensemble.py:115-154, common/model_based/utils.py:162-170; csrc/dyna.cu).
 *   out [E, N, 2*O] : raw output of the last EnsembleLayer (mean | logvar);  max_logvar / min_logvar [O]: the soft clamps (:118-119);
 *   model_idx [N]   : the elite model drawn for every row (np.random.choice(self.elites, N), :143 -- drawn on the host: RNG parity);
 *   noise [E, N, O] : standard normal draws (th.randn(std.shape), :128) or NULL = deterministic;
 *   obs [N, O - rew_dim] or NULL: added to the state part of the sample (the model predicts deltas, utils.py:165);
 *   sample_out / var_out [N, O]: sample and variance of the drawn model;  uncertainty_out [N]: sum_o sqrt(var_ensemble + 1e-12) (:146-149). */
MORL_API int morl_ensemble_sample_f32(const float* out, const float* max_logvar, const float* min_logvar, const int32_t* model_idx, const float* noise,
                                      const float* obs, int rew_dim, int E, int N, int O, float* sample_out, float* var_out, float* uncertainty_out,
                                      void* stream);
/* One imagined Dyna step, from the raw ensemble output to rows of the model replay buffer, in two launches (csrc/dyna.cu): the sample and
 * uncertainty of morl_ensemble_sample_f32 (same per-row arithmetic, same bits; obs always added), the termination rule, the uncertainty gate, the
 * ring append of the kept rows and the compaction of the alive rows (reference gpi_pd_continuous_action.py:346-366).
 *   out, max_logvar, min_logvar, model_idx, noise: as morl_ensemble_sample_f32;  obs [N, S], act [N, A]: the step's inputs, S = O - rew_dim;
 *   rule: MORL_TERM_* on (obs, act, s' = sample[rew_dim:], r = sample[:rew_dim]); a rule whose columns S / rew_dim lack is MORL_ERR_SHAPE;
 *   a row is kept iff uncertainty < max_uncertainty (strict: NaN is never kept);
 *   st_obs [capacity, S], st_next_obs [capacity, S], st_act [capacity, A], st_rew [capacity, rew_dim], st_done [capacity] (0.0 / 1.0): the ring,
 *     written as `kept` sequential adds starting at slot ptr would leave it (with kept > capacity only the last capacity rows; no slot twice);
 *   next_alive [N, S]: s' of the rows with done == 0, in row order;  uncertainty_out [N];  counts_out [2] = {kept, alive}, on the device.
 * Deterministic, no host synchronisation, capture-safe.  workspace: morl_dyna_commit_workspace_bytes(N) bytes, no initialisation required. */
#define MORL_TERM_NONE 0        /* halfcheetah, reacher, highway */
#define MORL_TERM_HOPPER 1      /* done unless s' finite, s'[1:] < 100, s'[0] > 0.7, |s'[1]| < 0.2 */
#define MORL_TERM_HUMANOID 2    /* done unless 1 < s'[0] < 2 */
#define MORL_TERM_MOUNTAINCAR 3 /* done iff s'[0] >= 0.45 and s'[1] >= 0 */
#define MORL_TERM_LUNARLANDER 4 /* done iff |s'[0]| >= 1, or r[0] != 0 and s'[6] >= 0.95 and s'[7] >= 0.95 */
MORL_API size_t morl_dyna_commit_workspace_bytes(int N);
MORL_API int morl_dyna_commit_f32(const float* out, const float* max_logvar, const float* min_logvar, const int32_t* model_idx, const float* noise,
                                  const float* obs, const float* act, int rew_dim, int E, int N, int O, int A, int rule, float max_uncertainty,
                                  float* st_obs, float* st_next_obs, float* st_act, float* st_rew, float* st_done, int capacity, int ptr,
                                  float* next_alive, float* uncertainty_out, int32_t* counts_out, void* workspace, void* stream);

/* Output layer of BOTH Q-networks + envelope operator + Bellman line as ONE kernel (csrc/qhead_envelope.cu): replaces, for the two no-grad
 * passes of Envelope.update (reference envelope.py:420, :429, :422-440, :298),
 *     morl_gemm_planes_f32 (online, N = A*D) + morl_gemm_planes_f32 (target) + morl_envelope_td_f32
 * -- the Q tensors live in registers / shared memory only (SURVEY 8(f)2: "envelope operator folded into the last-layer epilogue").
 *   a_on_planes / a_tg_planes : last hidden activations of the online / target net on s', planes [2][B*W][K] (row b*W + j), f16x2;
 *   w_on_planes / w_tg_planes : output-layer weight planes [2][32][K] (rows >= A*D zero), scales as in morl_gemm_planes_f32;
 *   everything from `wset` on  : as morl_envelope_td_f32 (same arithmetic contract, row orders, first-occurrence ties, outputs);
 *   q_on_out / q_tg_out        : optional fp32 copies of the Q tiles [B*W, A*D] (validation; NULL in the update).
 * The accumulation order equals morl_gemm_planes_f32's, so targets / indices are bit-identical to the three-launch chain.
 * morl_qhead_envelope_supported: 1 if the configuration is inside the kernel (f16x2 planes, W <= 64 dividing 128, B*W % 128 == 0,
 * A*D <= 32, W*A % 16 == 0, W*A*D % 4 == 0, 2 <= D <= 4, K % 64 == 0, K <= 256), else 0 -- callers then use the three-launch chain. */
MORL_API int morl_qhead_envelope_supported(int fmt, int B, int W, int A, int D, int K);
/* The kernel above without its operator half: the output layer of ONE network, q_out [M, N] = A . W^T + bias as fp32 rows (N <= 32: a narrow
 * morl_gemm_planes_f32 with the weight planes resident in shared memory and a deep activation ring; same accumulation order, bit-identical).
 * Used for the training pass's output layer (reference envelope.py:300).  M % 128 == 0, f16x2 planes, K % 64 == 0, K <= 256. */
MORL_API int morl_qhead_gemm_supported(int fmt, int M, int N, int K);
MORL_API int morl_qhead_gemm_f32(int fmt, const void* a_planes, long long a_plane_stride, const float* a_scale, const void* w_planes,
                                 long long w_plane_stride, const float* w_scale, const float* bias, int M, int N, int K, int reverse_tiles,
                                 float* q_out, void* stream);
MORL_API int morl_qhead_envelope_td_f32(int fmt, const void* a_on_planes, const void* a_tg_planes, long long a_plane_stride,
                                        const float* a_scale_on, const float* a_scale_tg, const void* w_on_planes, const void* w_tg_planes,
                                        long long w_plane_stride, const float* w_scale_on, const float* w_scale_tg, const float* bias_on,
                                        const float* bias_tg, int K, const float* wset, const float* reward, const float* done, float gamma,
                                        int B, int W, int A, int D, int dot_mode, int row_order, int reverse_tiles, float* target_out,
                                        int32_t* pref_out, int32_t* act_out, float* q_on_out, float* q_tg_out, void* stream);
/* h[b*W + j, :] = relu(u[b, :] + v[j, :]) written directly as planes [P][B*W][H] of scale * h (separable first layer of the
 * weight-conditioned Q-network: W1 [s || w] + b1 = W1_s s + (W1_w w + b1); reference envelope.py:75 builds the concat).
 * relu_bits_out (nullable): the ReLU bit mask of h in the layout of morl_gemm_planes_f32 ([B*W][8] words for H <= 256, [B*W][16] for
 * H <= 512; H % 32 == 0). */
MORL_API int morl_pairs_relu_split_planes(int fmt, const float* u, const float* v, int B, int W, int H, void* dst_planes,
                                          long long plane_stride, const float* scale, void* relu_bits_out, void* stream);

/* Product-conditioned first layer of GPI-PD's Q-network (reference gpi_pd.py:62-65, sf * wf):  h[b*P + p, :] = u[b, :] * v[p, :] (one fp32
 * multiply) written directly as planes [P_fmt][B*P][H] of scale * h.  u, v, dst 16-byte aligned, H % 8 == 0. */
MORL_API int morl_pairs_product_split_planes(int fmt, const float* u, const float* v, int B, int P, int H, void* dst_planes,
                                             long long plane_stride, const float* scale, void* stream);

/* Weight-gradient GEMM (reduction over the batch rows), split-K, deterministic:
 *   out[n, k] = sum_m G[m, n] * H[m, k]      G planes [P][M][ldg] (n < g_cols, scaled by *g_scale), H planes [P][M][ldh] (k < h_cols,
 *   scaled by *h_scale);  ldg, ldh multiples of 64, ldh <= 512;  transpose_out != 0 stores out[k, n] instead.  Replaces the
 *   dW = dY^T X products that torch autograd issues for the nn.Linear layers of the reference networks (loss.backward(), envelope.py:316).
 *   colsum_out (nullable, [g_cols]): out_b[n] = sum_m G[m, n], the bias gradient db = colsum(dY), evaluated in the same pass as
 *   G^T . ones on the tensor cores (replaces a separate sweep of the G planes).
 *   workspace: morl_gemm_mn_workspace_bytes(M, g_cols, h_cols) bytes. */
MORL_API size_t morl_gemm_mn_workspace_bytes(int M, int a_cols, int b_cols);
MORL_API int morl_gemm_planes_mn_f32(int fmt, const void* g_planes, long long g_plane_stride, int ldg, int g_cols, const float* g_scale,
                                     const void* h_planes, long long h_plane_stride, int ldh, int h_cols, const float* h_scale, int M,
                                     int transpose_out, float* out, int ld_out, float* colsum_out, void* workspace, void* stream);
/* gradients of the separable first layer: dU[b,:] = sum_j G[b*W+j,:], dV[j,:] = sum_b G[b*W+j,:]  (G planes [P][B*W][H] scaled by
 * *scale, W <= 64 for the one-pass kernel); workspace: morl_pairs_grad_reduce_workspace_bytes(B, W, H) bytes */
MORL_API size_t morl_pairs_grad_reduce_workspace_bytes(int B, int W, int H);
MORL_API int morl_pairs_grad_reduce_planes(int fmt, const void* planes, long long plane_stride, const float* scale, int B, int W, int H,
                                           float* dU, float* dV, void* workspace, void* stream);

/* Separable first layer of the weight-conditioned Q-network on the pair batch (reference envelope.py:59-77 builds [s || w] rows for
 * nn.Linear; DESIGN.md section 2):  u[b, :] = W1[:, :F] feats[b],  v[j, :] = W1[:, F:] wset[j] + b1  in ONE launch (replaces two library
 * sgemms and their epilogue kernels).  W1 is the row-major nn.Linear weight [H, F + D]; u [B, H], v [W, H]. */
MORL_API int morl_pair_layer1_uv_f32(const float* feats, const float* wset, const float* W1, const float* b1, int B, int W, int F, int D, int H,
                                     float* u, float* v, void* stream);

/* The two feature maps of GPI-PD's Q-network in ONE launch:  u = relu(s . Ls^T + bs) [B, H] (state_features on the B observations s [B, F])
 * and v = relu(m . Lw^T + bw) [P, H] (weights_features on the P weight vectors m [P, D]); Ls [H, F], Lw [H, D] row-major nn.Linear weights. */
MORL_API int morl_product_layer1_uv_f32(const float* s, const float* Ls, const float* bs, int B, int F, const float* m, const float* Lw, const float* bw,
                                        int P, int D, int H, float* u, float* v, void* stream);

/* Parameter gradients of the separable first layer (backward of morl_pair_layer1_uv_f32; autograd of nn.Linear at envelope.py:316 on the
 * effective batch, restricted to layer 1):  dW1 [H, F + D] = [dU^T feats | dV^T wset],  db1 [H] = colsum(dV), with dU [B, H] / dV [W, H]
 * from morl_pairs_grad_reduce_planes.  One launch, deterministic split reduction.  `workspace`: morl_pair_layer1_grad_workspace_bytes(F, D,
 * H) bytes that must be ZERO before the first call (the kernel leaves its arrival counters zeroed again). */
MORL_API size_t morl_pair_layer1_grad_workspace_bytes(int F, int D, int H);
MORL_API int morl_pair_layer1_grad_f32(const float* dU, const float* dV, const float* feats, const float* wset, int B, int W, int F,
                              int D, int H, float* dW1, float* db1, void* workspace, void* stream);


/* Fused gradient clipping + Adam step over a list of tensors (two launches).  Replaces th.nn.utils.clip_grad_norm_ +
 * optim.Adam.step (envelope.py:324-326; torch/optim/adam.py _single_tensor_adam arithmetic, amsgrad = False, weight_decay = 0).
 *   params/grads/exp_avg/exp_avg_sq/steps : device arrays of n_tensors device pointers (steps[t] -> float32 scalar, incremented here)
 *   max_grad_norm <= 0 disables clipping;  workspace: morl_adam_workspace_bytes(n_tensors, max_size) bytes */
MORL_API size_t morl_adam_workspace_bytes(int n_tensors, int64_t max_size);
MORL_API int morl_adam_clip_f32(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                                float* const* steps, const int64_t* sizes, int n_tensors, int64_t max_size, float max_grad_norm,
                                float lr, float beta1, float beta2, float eps, void* workspace, void* stream);
/* morl_adam_clip_lr_f32: the same step with the learning rate read at run time from the device double *lr (a CUDA graph captured once
 * follows a learning-rate schedule); step_size = (float)(*lr / (1 - beta1^t)) as Python forms it from a float lr. */
MORL_API int morl_adam_clip_lr_f32(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                                   float* const* steps, const int64_t* sizes, int n_tensors, int64_t max_size, float max_grad_norm,
                                   const double* lr, float beta1, float beta2, float eps, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MO-PPO (reference single_policy/ser/mo_ppo.py), csrc/ppo.cu.
 *
 * morl_vector_gae_f32 (:439-476): rewards, values f32 [T, E, D], dones f32 [T, E], next_value f32 [E, D], next_done f32 [E],
 *   weights f32 [D].  With nnt_t = 1 - dones[t + 1] (1 - next_done for t = T - 1) and nv_t = values[t + 1] (next_value for T - 1),
 *   every operation rounded once, in the reference's order (g = (float)gamma, gl = (float)(gamma * gae_lambda)):
 *     use_gae = 1: delta = (r + (g * nv) * nnt) - v;  lastgaelam = delta + (gl * nnt) * lastgaelam  (0 before the last step);
 *                  returns = lastgaelam + v;  advantage vector = lastgaelam
 *     use_gae = 0: returns[t] = r + (g * nnt) * returns[t + 1]  (next_value for T - 1);  advantage vector = returns - v
 *   so returns [T, E, D] are bit-exact against the reference.  advantages [T, E] = advantage vector . weights, summed in double and
 *   rounded once (the reference's matmul may round differently).  D <= MORL_MAX_D.
 *
 * morl_ppo_loss_f32 (:514-549): one minibatch of M rows in ONE CTA.  mean f32 [M, A] (actor output), logstd f32 [A], value f32 [M, D]
 *   (critic output), actions [M, A], old_logprob [M], advantages [M] (raw, scalarised), returns and old_values [M, D] (old_values
 *   may be NULL without clip_vloss).  sigma = exp(logstd); logp = sum_j Normal(mean, sigma).log_prob(action); ratio = exp(logp - old);
 *   advantages normalised by torch's unbiased std() + 1e-8 when norm_adv (refused for M < 2); pg_loss = mean max(-adv ratio,
 *   -adv clamp(ratio, 1 -+ clip)); v_loss = 0.5 mean over M*D of (v - R)^2, or of max((v - R)^2, (clip(v) - R)^2) with clip_vloss;
 *   entropy = sum_j (0.5 + 0.5 log 2pi + logstd_j);  loss_out[0] = pg_loss - ent_coef * entropy + v_loss * vf_coef.
 *   dmean [M, A], dlogstd [A], dvalue [M, D]: d loss_out / d input, with torch's backward rules: th.max splits the gradient half and
 *   half on a tie, clamp passes it on its closed interval.  stats f32 [6]: pg_loss, v_loss, entropy, old_approx_kl, approx_kl are
 *   written; stats[5] += the clip fraction (a sum over the minibatches of an update; zero it before the first).  Reductions are fixed
 *   block trees in double (deterministic).  A <= 32, D <= MORL_MAX_D. */
MORL_API int morl_vector_gae_f32(const float* rewards, const float* values, const float* dones, const float* next_value, const float* next_done,
                                 const float* weights, int T, int E, int D, double gamma, double gae_lambda, int use_gae, float* returns,
                                 float* advantages, void* stream);
/* morl_vector_gae_objectives_f32 (nl_mo_ppo.py:290-308): the use_gae = 1 recursion of morl_vector_gae_f32 with the same rounding, writing the
 *   per-objective advantages [T, E, D] (lastgaelam) instead of their weighted sum; returns [T, E, D] as there.  D <= MORL_MAX_D. */
MORL_API int morl_vector_gae_objectives_f32(const float* rewards, const float* values, const float* dones, const float* next_value,
                                            const float* next_done, int T, int E, int D, double gamma, double gae_lambda, float* returns,
                                            float* advantages, void* stream);
MORL_API int morl_ppo_loss_f32(const float* mean, const float* logstd, const float* value, const float* actions, const float* old_logprob,
                               const float* advantages, const float* returns, const float* old_values, int M, int A, int D, float clip_coef,
                               float ent_coef, float vf_coef, int norm_adv, int clip_vloss, float* loss_out, float* dmean, float* dlogstd,
                               float* dvalue, float* stats, void* stream);

/* ------------------------------------------------------------------------------------------------
 * PCN / LCN (reference multi_policy/pcn/pcn.py, multi_policy/lcn/lcn.py), csrc/pcn.cu.
 *
 * The default model (pcn.py:51-103): c = [desired_return || horizon] * scaling [d + 1], s = sigmoid(Ls obs + bs),
 *   e = sigmoid(Lc c + bc), h = relu(W1 (s * e) + b1), y = W2 h + b2; log_softmax(y) for discrete actions, y for continuous ones.
 *   params / grads: HOST arrays of 8 device pointers, in state-dict order: Ls [H, S], bs [H], Lc [H, d + 1], bc [H], W1 [H, H], b1 [H],
 *   W2 [A, H], b2 [A] (A = number of actions, or the action dimension when continuous).
 * Supported range (morl_pcn_supported): 1 <= S <= 256, 1 <= d <= MORL_MAX_D, H in {32, 64, 128, 256}, 1 <= A <= 32, and for the update
 *   1 <= B <= MORL_PCN_MAX_BATCH; anything else returns MORL_ERR_UNSUPPORTED.
 *
 * morl_pcn_update_f32 (pcn.py:202-236): one minibatch gathered from the episode store, f32 [N, ld_store] with the columns
 *   [obs (S) | return-to-go (d) | action]; the action is one int32 (its bits stored in the f32 column) for discrete actions, A floats
 *   for continuous ones.  Row b of the batch reads store row rows[b] (obs, desired return = return-to-go, action) and horizon = horizons[b].
 *   loss_out[0] = mean over rows of -log_softmax(y)[a] (discrete) or mse_loss(action, y) (continuous); entropy_out[0] (discrete, nullable)
 *   = sum over the batch of -exp(lp) lp; pred_out (nullable) [B, A] = the log-probabilities or predictions.  grads[t] are OVERWRITTEN with
 *   d loss / d params[t].  Deterministic: per-tile partials over 16 rows in row order, then a fixed-order sum over the tiles (no float
 *   atomics), so repeated launches and graph replays are bit-identical.  Two launches.  workspace: morl_pcn_workspace_bytes(...) bytes.
 * morl_pcn_forward_f32 (pcn.py:309-322): the forward on N rows with their own commands: obs [N, S], ret [N, d], hor [N] -> out [N, A]
 *   (log-probabilities when log_softmax, else predictions); argmax_out (nullable) int32 [N] = first index of the row maximum.  obs, ret,
 *   hor, out and argmax_out may be pinned host memory (read and written through unified addressing).  One launch. */
#define MORL_PCN_MAX_BATCH 4096
MORL_API int morl_pcn_supported(int obs_dim, int d, int hidden, int n_out, int batch);
MORL_API size_t morl_pcn_workspace_bytes(int obs_dim, int d, int hidden, int n_out, int batch);
MORL_API int morl_pcn_update_f32(const float* const* params, float* const* grads, const float* scaling, const float* store, int ld_store,
                                 const int32_t* rows, const int32_t* horizons, int B,
                                 int obs_dim, int d, int hidden, int n_out, int continuous, float* loss_out, float* entropy_out,
                                 float* pred_out, void* workspace, void* stream);
MORL_API int morl_pcn_forward_f32(const float* const* params, const float* scaling, const float* obs, const float* ret, const float* hor, int N,
                                  int obs_dim, int d, int hidden, int n_out, int log_softmax, float* out, int32_t* argmax_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * EUPG (reference single_policy/esr/eupg.py), csrc/eupg.cu.
 *
 * The policy network (eupg.py:22-75): x = [obs (S) || accrued reward (d)], hidden layers a = tanh(W a + b) of widths hidden[0..n_hidden-1],
 *   logits z = W_L a + b_L [A], p = sigmoid(z) / sum_a sigmoid(z_a) per row, log p_a = log(clamp(p_a, 2^-23, 1 - 2^-23)) (no gradient
 *   where the clamp acts).  params / grads: HOST arrays of 2 (n_hidden + 1) device pointers in state-dict order: W_0 [h_0, S + d], b_0,
 *   ..., W_L [A, h_last], b_L [A].  hidden: HOST int array [n_hidden].
 * Supported range (morl_eupg_supported, no device needed): 1 <= S, 1 <= d <= MORL_MAX_D, S + d <= 256, 1 <= n_hidden <= 4, every width in
 *   [1, 256], 1 <= A <= 32; anything else returns MORL_ERR_UNSUPPORTED.
 *
 * morl_eupg_returns_f32 (eupg.py:263-270): out [T, d] = discounted forward returns of rewards [T, d] (row stride ld floats), c = gamma * c + r_t
 *   from t = T - 1 down to 0, product and sum rounded separately in float32: bit-identical to the reference's loop.  Any d >= 1 (it is not
 *   limited to MORL_MAX_D: objectives are independent).  out: contiguous [T, d].  One launch.
 * morl_eupg_update_f32 (eupg.py:226-251): one episode of T rows, row t reading obs int32 [S] at obs + t * ld, the accrued reward f32 [d] at
 *   acc + t * ld and the action int32 (in [0, A)) at actions + t * ld (one interleaved staging block), and v[t * v_stride] (v_stride >= 0;
 *   0 broadcasts one value).  loss_out[0] = -mean_t(log p_{action_t} * v_t); grads[t] are OVERWRITTEN with d loss / d params[t].
 *   Deterministic: a fixed number of CTAs folds contiguous ranges of 16-row tiles in order, then a fixed-order sum over the CTAs (no float
 *   atomics); results depend on neither the SM count nor the run.  Two launches.  workspace: morl_eupg_workspace_bytes(...) bytes, which do
 *   not depend on T.
 * morl_eupg_probs_f32 (eupg.py:46-61): p [N, A] of rows x [N, S + d]; x and out may be pinned host memory.  One launch. */
MORL_API int morl_eupg_supported(int obs_dim, int d, const int* hidden, int n_hidden, int n_out);
MORL_API size_t morl_eupg_workspace_bytes(int obs_dim, int d, const int* hidden, int n_hidden, int n_out);
MORL_API int morl_eupg_returns_f32(const float* rewards, int ld, int T, int d, float gamma, float* out, void* stream);
MORL_API int morl_eupg_update_f32(const float* const* params, float* const* grads, const int32_t* obs, const float* acc, const int32_t* actions,
                                  int ld, const float* v, int v_stride, int T, int obs_dim, int d, const int* hidden, int n_hidden, int n_out,
                                  float* loss_out, void* workspace, void* stream);
MORL_API int morl_eupg_probs_f32(const float* const* params, const float* x, int N, int obs_dim, int d, const int* hidden, int n_hidden,
                                 int n_out, float* out, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Non-linear MO-PPO (reference single_policy/ser/nl_mo_ppo.py), csrc/nl_ppo.cu.
 *
 * The reference's Agent (nl_mo_ppo.py:26-108): x = [obs (S) || accrued reward (d) || pref (Dp)] with Dp in {0, d} (pref: one device vector
 *   [Dp] shared by every row; zeros when the learner has no preference), critic x -> tanh(64) -> tanh(64) -> d, actor x -> tanh(64) ->
 *   tanh(64) -> A logits of a Categorical.  params / grads: HOST arrays of the 12 device pointers in the Agent's parameter order
 *   (critic.0.weight [64, K], critic.0.bias, critic.2.weight [64, 64], critic.2.bias, critic.4.weight [d, 64], critic.4.bias, then the
 *   same six of the actor with actor.4.weight [A, 64]); K = S + d + Dp.
 * Supported range (morl_nl_ppo_supported, no device needed): 1 <= S, 1 <= d <= MORL_MAX_D, Dp in {0, d}, K <= 256, 1 <= A <= 32 and a
 *   minibatch (batch) of 1 to 4096 rows; anything else returns MORL_ERR_UNSUPPORTED.
 *
 * morl_nl_ppo_update_f32 (nl_mo_ppo.py:344-393): one minibatch of M rows; row i is source row perm[i] (int64) of obs f32 [B, S],
 *   acc f32 [B, d], actions int64 [B], old_logprob [B], advantages / returns / old_values f32 [B, d] (old_values may be NULL without
 *   clip_vloss).  With norm_adv (refused for M < 2) each objective's advantages are normalised by their minibatch mean and unbiased std
 *   + 1e-8.  pg_loss = sum_o w_o mean_i max(-adv_io r_i, -adv_io clamp(r_i, 1 -+ clip)), r = exp(logp - old); v_loss = 0.5 mean over M*d of
 *   (v - R)^2 or, with clip_vloss, of max((v - R)^2, (clip(v) - R)^2); entropy = mean Categorical entropy;
 *   loss_out[0] (nullable) = pg_loss - ent_coef * entropy + vf_coef * v_loss.  grads are OVERWRITTEN with d loss / d params, with torch's
 *   backward rules (th.max splits a tie half and half, clamp passes on its closed interval).  stats f32 [6]: pg_loss, v_loss, entropy,
 *   old_approx_kl, approx_kl written; stats[5] += the clip fraction.  loss_weights f32 [d] is read at run time.  A fixed number of CTAs each
 *   folds a contiguous range of 16-row tiles into its own partial, a second launch sums them in CTA order: no float atomics, results depend
 *   on neither the SM count nor the run.  workspace: morl_nl_ppo_workspace_bytes(...) bytes, independent of M.  Two launches.
 * morl_nl_ppo_forward_f32 (nl_mo_ppo.py:90-108): rows [obs (N x S) || acc (N x d) || pref]; logits [N, A], values [N, d] and argmax_out int32
 *   [N] (first occurrence of the row maximum) are each nullable, at least one given.  obs, acc and the outputs may be pinned host memory.
 *   One launch.
 * morl_nl_ppo_commit_f32 (nl_mo_ppo.py:251-275): one rollout step of E environments.  For each e: row `step` of obs_store [T, E, S],
 *   acc_store [T, E, d] and done_store [T, E] takes the carried next_obs [E, S], next_acc [E, d] and next_done [E]; act_store int64 [T, E]
 *   takes action[e]; logp_store [T, E] the log-softmax of logits [E, A] at it; rew_store [T, E, d] the staged reward.  staged f32
 *   [E, S + d + 2] = obs | reward | terminated | truncated of the environment step; then next_obs = obs, next_done = terminated | truncated,
 *   next_acc = (next_acc + powf((float)gamma, (float)t) * reward) * (1 - next_done) and timestep int32 [E] t = (t + 1) * (1 - next_done),
 *   each operation rounded once as torch's device expression.  One launch. */
MORL_API int morl_nl_ppo_supported(int obs_dim, int d, int pref_dim, int n_actions, int batch);
MORL_API size_t morl_nl_ppo_workspace_bytes(int obs_dim, int d, int pref_dim, int n_actions);
MORL_API int morl_nl_ppo_update_f32(const float* const* params, float* const* grads, const float* obs, const float* acc, const int64_t* actions,
                                    const float* old_logprob, const float* advantages, const float* returns, const float* old_values,
                                    const int64_t* perm, int M, int obs_dim, int d, int pref_dim, int n_actions, const float* pref,
                                    const float* loss_weights, float clip_coef, float ent_coef, float vf_coef, int norm_adv, int clip_vloss,
                                    float* loss_out, float* stats, void* workspace, void* stream);
MORL_API int morl_nl_ppo_forward_f32(const float* const* params, const float* obs, const float* acc, int N, int obs_dim, int d, int pref_dim,
                                     int n_actions, const float* pref, float* logits, float* values, int32_t* argmax_out, void* stream);
MORL_API int morl_nl_ppo_commit_f32(const float* staged, const float* logits, const int64_t* action, int step, int E, int obs_dim, int d,
                                    int n_actions, double gamma, float* obs_store, float* acc_store, float* done_store, float* rew_store,
                                    int64_t* act_store, float* logp_store, float* next_obs, float* next_acc, float* next_done, int32_t* timestep,
                                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MORL_B200_H_ */
