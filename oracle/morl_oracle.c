/*
 * morl_oracle.c -- TEST INFRASTRUCTURE ONLY.  Plain-C CPU restatement of the reference algorithms on the hot path
 * (LucasAlegre/morl-baselines @ a8acdbb).  It is the checker for the CUDA kernels: only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path never does.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC (see oracle/Makefile); contraction is disabled so that
 * every a*b+c below is two IEEE roundings unless fmaf() is written explicitly.
 *
 * PARITY PINNING: the reference's own tests hold known-answer vectors only for the Pareto prune
 * (tests/test_pruning.py:68-128); those are reproduced in tests/test_pareto_oracle.py.  Everything else is pinned
 * against outputs of the unmodified reference run in the build container (tests/golden/make_golden.py ->
 * tests/golden/ *.npz), see DESIGN.md "Oracle".
 *
 * Each function cites the reference lines it restates (paths relative to the reference root).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define DOT_UNFUSED 0
#define DOT_FMA 1
#define DOT_PAIRFMA 2
#define MAP_TILE 0
#define MAP_BLOCK 1
#define ROWS_REFERENCE 0
#define ROWS_BMAJOR 1

/* scalarisation w . q; the three arithmetics documented in include/morl_b200.h */
static float dotw(const float* w, const float* q, int D, int mode) {
    if (mode == DOT_UNFUSED) {
        float acc = w[0] * q[0];
        for (int r = 1; r < D; ++r) {
            float p = w[r] * q[r];
            acc = acc + p;
        }
        return acc;
    } else if (mode == DOT_FMA) {
        float acc = w[0] * q[0];
        for (int r = 1; r < D; ++r) acc = fmaf(w[r], q[r], acc);
        return acc;
    } else {
        float acc = 0.f;
        int r = 0;
        for (; r + 1 < D; r += 2) {
            float p0 = w[r] * q[r];
            float p = fmaf(w[r + 1], q[r + 1], p0);
            acc = (r == 0) ? p : acc + p;
        }
        if (D % 2 == 1) {
            float t = w[D - 1] * q[D - 1];
            acc = (D == 1) ? t : acc + t;
        }
        return acc;
    }
}

/* envelope.py:298  target_q = b_rewards + (1 - b_dones) * self.gamma * target   (three separate elementwise ops) */
static float bellman(float r, float done, float gamma, float q) {
    float nd = 1.0f - done;
    nd = nd * gamma;
    float t = nd * q;
    return r + t;
}

static int map_row(int k, int rows, int n, int map) {
    if (rows == n) return k;
    if (rows == 1) return 0;
    return map == MAP_TILE ? (k % rows) : (k / (n / rows));
}

/* Envelope.envelope_target, multi_policy/envelope/envelope.py:404-440, + the Bellman line :298.
 * Restated in the reference's own two-stage form: th.max over actions (dim=2, first occurrence), then th.argmax over
 * sampled weights (dim=1, first occurrence), then the two gathers from the TARGET net -- on the B*W distinct rows
 * (the reference's B*W^2 tiling repeats each (s'_b, w_j) row W times; identical values, SURVEY.md headline 2). */
void oracle_envelope_td(const float* q_on, const float* q_tg, const float* wset, const float* reward, const float* done,
                        float gamma, int B, int W, int A, int D, int mode, int row_order, float* target, int32_t* pref,
                        int32_t* act) {
    for (int i = 0; i < W; ++i) {
        const float* w = wset + (size_t)i * D;
        for (int b = 0; b < B; ++b) {
            float best_j_val = 0.f;
            int best_j = 0, best_a_of_best_j = 0;
            for (int j = 0; j < W; ++j) {
                /* max_q[j], ac[j] = th.max(scalarized[k, j, :]) */
                float mval = 0.f;
                int marg = 0;
                for (int a = 0; a < A; ++a) {
                    float s = dotw(w, q_on + (((size_t)b * W + j) * A + a) * D, D, mode);
                    if (a == 0 || s > mval) {
                        mval = s;
                        marg = a;
                    }
                }
                /* pref = th.argmax(max_q) */
                if (j == 0 || mval > best_j_val) {
                    best_j_val = mval;
                    best_j = j;
                    best_a_of_best_j = marg;
                }
            }
            size_t k = (row_order == ROWS_REFERENCE) ? ((size_t)i * B + b) : ((size_t)b * W + i);
            const float* qt = q_tg + (((size_t)b * W + best_j) * A + best_a_of_best_j) * D;
            for (int r = 0; r < D; ++r) target[k * D + r] = bellman(reward[(size_t)b * D + r], done[b], gamma, qt[r]);
            if (pref) pref[k] = best_j;
            if (act) act[k] = best_a_of_best_j;
        }
    }
}

/* The three per-row targets below take the first argmax with a strict `>` from -inf, as the kernels do
 * (include/morl_b200.h): a NaN score never wins, and a row whose every score is -inf or NaN falls back to candidate 0.
 * th.argmax would return the first NaN instead; the two differ only on rows with a NaN score. */

/* Envelope.ddqn_target, envelope.py:442-463 (+ :298 when reward != NULL); GPIPD._reset_priorities non-GPI branch gpi_pd.py:648-656 */
void oracle_greedy_td(const float* q_sel, const float* q_eval, const float* w, int w_rows, int w_map, const float* reward,
                      const float* done, int r_rows, int r_map, float gamma, int N, int A, int D, int mode, float* out,
                      int32_t* act) {
    for (int k = 0; k < N; ++k) {
        const float* wv = w + (size_t)map_row(k, w_rows, N, w_map) * D;
        float mval = -INFINITY;
        int marg = -1;
        for (int a = 0; a < A; ++a) {
            float s = dotw(wv, q_sel + ((size_t)k * A + a) * D, D, mode);
            if (s > mval) {
                mval = s;
                marg = a;
            }
        }
        if (marg < 0) marg = 0; /* every score -inf or NaN */
        const float* qe = q_eval + ((size_t)k * A + marg) * D;
        if (reward) {
            int ri = map_row(k, r_rows, N, r_map);
            for (int r = 0; r < D; ++r) out[(size_t)k * D + r] = bellman(reward[(size_t)ri * D + r], done[ri], gamma, qe[r]);
        } else {
            for (int r = 0; r < D; ++r) out[(size_t)k * D + r] = qe[r];
        }
        if (act) act[k] = marg;
    }
}

/* GPIPD.update target block, multi_policy/gpi_pd/gpi_pd.py:445-463: th.argmin over the stacked target nets of the
 * scalarised values (first occurrence), gather, then greedy action of the gathered values, gather, Bellman. */
void oracle_critic_min_td(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map, const float* reward,
                          const float* done, int r_rows, int r_map, float gamma, int N, int A, int D, int mode, float* out,
                          int32_t* act) {
    size_t stride = (size_t)N * A * D;
    for (int k = 0; k < N; ++k) {
        const float* wv = w + (size_t)map_row(k, w_rows, N, w_map) * D;
        float best = -INFINITY;
        int ba = -1, bn = 0;
        for (int a = 0; a < A; ++a) {
            float smin = 0.f;
            int nmin = 0;
            for (int n = 0; n < n_nets; ++n) {
                float s = dotw(wv, q_nets + n * stride + ((size_t)k * A + a) * D, D, mode);
                if (n == 0 || s < smin) {
                    smin = s;
                    nmin = n;
                }
            }
            if (a == 0) bn = nmin;
            /* max_q = einsum(w, gathered) recomputes the same scalarisation of the selected net */
            if (smin > best) {
                best = smin;
                ba = a;
                bn = nmin;
            }
        }
        if (ba < 0) ba = 0; /* every score -inf or NaN: action 0 with its critic-min net */
        const float* qe = q_nets + bn * stride + ((size_t)k * A + ba) * D;
        if (reward) {
            int ri = map_row(k, r_rows, N, r_map);
            for (int r = 0; r < D; ++r) out[(size_t)k * D + r] = bellman(reward[(size_t)ri * D + r], done[ri], gamma, qe[r]);
        } else {
            for (int r = 0; r < D; ++r) out[(size_t)k * D + r] = qe[r];
        }
        if (act) act[k] = ba;
    }
}

/* GPIPD._envelope_target gpi_pd.py:662-690; gpi_action gpi_pd.py:564-582 (n_nets=1, no Bellman);
 * GPIPDContinuousAction.eval GPI branch gpi_pd_continuous_action.py:464-478. Two-stage (max over a, argmax over p). */
void oracle_gpi_envelope(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map, const float* reward,
                         const float* done, int r_rows, int r_map, float gamma, int B, int P, int A, int D, int mode,
                         float* out, int32_t* policy, int32_t* act) {
    size_t stride = (size_t)B * P * A * D;
    for (int b = 0; b < B; ++b) {
        const float* wv = w + (size_t)map_row(b, w_rows, B, w_map) * D;
        float bestp = -INFINITY;
        int bp = -1, bpa = 0, bpn = 0, n00 = 0;
        for (int p = 0; p < P; ++p) {
            float besta = -INFINITY;
            int ba = 0, bn = 0;
            for (int a = 0; a < A; ++a) {
                float smin = 0.f;
                int nmin = 0;
                for (int n = 0; n < n_nets; ++n) {
                    float s = dotw(wv, q_nets + n * stride + ((((size_t)b * P + p) * A) + a) * D, D, mode);
                    if (n == 0 || s < smin) {
                        smin = s;
                        nmin = n;
                    }
                }
                if (p == 0 && a == 0) n00 = nmin;
                if (smin > besta) {
                    besta = smin;
                    ba = a;
                    bn = nmin;
                }
            }
            if (besta > bestp) {
                bestp = besta;
                bp = p;
                bpa = ba;
                bpn = bn;
            }
        }
        if (bp < 0) { /* every score -inf or NaN: candidate (0, 0) with its critic-min net */
            bp = 0;
            bpa = 0;
            bpn = n00;
        }
        const float* qe = q_nets + bpn * stride + ((((size_t)b * P + bp) * A) + bpa) * D;
        if (out) {
            if (reward) {
                int ri = map_row(b, r_rows, B, r_map);
                for (int r = 0; r < D; ++r) out[(size_t)b * D + r] = bellman(reward[(size_t)ri * D + r], done[ri], gamma, qe[r]);
            } else {
                for (int r = 0; r < D; ++r) out[(size_t)b * D + r] = qe[r];
            }
        }
        if (policy) policy[b] = bp;
        if (act) act[b] = bpa;
    }
}

/* capql.py:326-331 (variant 0), mosac_continuous_action.py:435-442 (variant 1), gpi_pd_continuous_action.py:395-403 (variant 2) */
void oracle_actor_critic_td(const float* q_nets, int n_nets, const float* w, int w_rows, int w_map, const float* reward,
                            const float* done, const float* logp, float alpha, float gamma, int N, int D, int variant,
                            float* out) {
    size_t stride = (size_t)N * D;
    for (int k = 0; k < N; ++k) {
        const float* wv = (variant == 0) ? NULL : w + (size_t)map_row(k, w_rows, N, w_map) * D;
        float ent = logp ? alpha * logp[k] : 0.f;
        if (variant == 0) {
            for (int r = 0; r < D; ++r) {
                float m = q_nets[(size_t)k * D + r];
                for (int n = 1; n < n_nets; ++n) {
                    float v = q_nets[n * stride + (size_t)k * D + r];
                    if (v < m) m = v;
                }
                float soft = m - ent;
                out[(size_t)k * D + r] = bellman(reward[(size_t)k * D + r], done[k], gamma, soft);
            }
        } else if (variant == 1) {
            float m = 0.f;
            for (int n = 0; n < n_nets; ++n) {
                float s = dotw(wv, q_nets + n * stride + (size_t)k * D, D, DOT_UNFUSED);
                if (n == 0 || s < m) m = s;
            }
            float rs = dotw(wv, reward + (size_t)k * D, D, DOT_UNFUSED);
            float soft = m - ent;
            out[k] = bellman(rs, done[k], gamma, soft);
        } else {
            float smin = 0.f;
            int nmin = 0;
            for (int n = 0; n < n_nets; ++n) {
                float s = dotw(wv, q_nets + n * stride + (size_t)k * D, D, DOT_UNFUSED);
                if (n == 0 || s < smin) {
                    smin = s;
                    nmin = n;
                }
            }
            for (int r = 0; r < D; ++r) {
                float qv = q_nets[nmin * stride + (size_t)k * D + r] - ent;
                out[(size_t)k * D + r] = bellman(reward[(size_t)k * D + r], done[k], gamma, qv);
            }
        }
    }
}

/* envelope.py:301-313 (gather, mse_loss, homotopy auxiliary loss) and :329-331 (priorities of weight index 0);
 * loss accumulated in double (the tolerance against torch's float reduction is stated in the tests) */
void oracle_td_mse(const float* q_values, const int32_t* action, const float* target_q, const float* wset, float lambda,
                   int B, int W, int A, int D, int row_order, float* loss_out, float* grad_q, float* q_taken, float* prio) {
    long long N = (long long)B * W;
    double sq = 0.0, aux2 = 0.0;
    if (grad_q) memset(grad_q, 0, sizeof(float) * (size_t)N * A * D);
    for (long long k = 0; k < N; ++k) {
        int i, b;
        if (row_order == ROWS_REFERENCE) {
            i = (int)(k / B);
            b = (int)(k % B);
        } else {
            b = (int)(k / W);
            i = (int)(k % W);
        }
        int a = action[b];
        const float* q = q_values + ((size_t)k * A + a) * D;
        const float* t = target_q + (size_t)k * D;
        const float* w = wset + (size_t)i * D;
        float d[8];
        for (int r = 0; r < D; ++r) {
            d[r] = q[r] - t[r];
            sq += (double)d[r] * (double)d[r];
        }
        float aux = 0.f;
        if (lambda > 0.f) {
            aux = dotw(q, w, D, DOT_UNFUSED) - dotw(t, w, D, DOT_UNFUSED);
            aux2 += (double)aux * (double)aux;
        }
        if (q_taken)
            for (int r = 0; r < D; ++r) q_taken[(size_t)k * D + r] = q[r];
        if (grad_q) {
            double c1 = (1.0 - (double)lambda) * 2.0 / ((double)N * D);
            double c2 = (double)lambda * 2.0 / (double)N;
            for (int r = 0; r < D; ++r) grad_q[((size_t)k * A + a) * D + r] = (float)(c1 * d[r] + c2 * aux * w[r]);
        }
        if (prio && i == 0) prio[b] = fabsf(dotw(d, w, D, DOT_UNFUSED));
    }
    double mse = sq / ((double)N * D), auxl = aux2 / (double)N;
    loss_out[0] = (float)((lambda > 0.f) ? ((1.0 - lambda) * mse + lambda * auxl) : mse);
}

/* gpi_pd.py:469-487 with common/networks.py:90-100 (huber) and gpi_pd.py:507-520 (raw |w . max_n err| priorities) */
void oracle_td_huber(const float* q_values, int n_nets, const int32_t* action, int a_rows, const float* target_q,
                     const float* target_gpi, const float* w, int w_rows, int w_map, float min_priority, int N, int A, int D,
                     int p_rows, float* loss_out, float* grad_q, float* prio) {
    size_t stride = (size_t)N * A * D;
    double lsum = 0.0;
    if (grad_q) memset(grad_q, 0, sizeof(float) * stride * n_nets);
    for (int k = 0; k < N; ++k) {
        int a = action[k % a_rows];
        float emax[8];
        for (int n = 0; n < n_nets; ++n) {
            for (int r = 0; r < D; ++r) {
                float q = q_values[n * stride + ((size_t)k * A + a) * D + r];
                float d = q - target_q[(size_t)k * D + r];
                float x = fabsf(d);
                lsum += (x < min_priority) ? 0.5 * (double)x * x : (double)min_priority * x;
                if (grad_q) {
                    double g = (x < min_priority) ? d : (d > 0 ? min_priority : (d < 0 ? -min_priority : 0.0));
                    grad_q[n * stride + ((size_t)k * A + a) * D + r] = (float)(g / ((double)N * D) / n_nets);
                }
                float e = target_gpi ? fabsf(q - target_gpi[(size_t)k * D + r]) : x;
                emax[r] = (n == 0 || e > emax[r]) ? e : emax[r];
            }
        }
        if (prio && k < p_rows) {
            const float* wv = w + (size_t)map_row(k, w_rows, N, w_map) * D;
            prio[k] = fabsf(dotw(wv, emax, D, DOT_UNFUSED));
        }
    }
    loss_out[0] = (float)(lsum / ((double)N * D) / n_nets);
}

/* get_non_pareto_dominated_inds, common/pareto.py:34-57, restated from its own definition:
 *   counts[invs][i] = multiplicity of row i's value (np.unique(axis=0, return_counts))
 *   c1[i] = #{j : pts[j] >= pts[i] in every coordinate} == multiplicity(i)      (res_eq, :47, :49)
 *   c2[i] = exists j with NOT(pts[j] > pts[i] in every coordinate)              (res_g, :48, :50)
 *   to_keep[i] = i is the first index of its value (np.unique return_index)      (:51-53)
 * Generic over float / double via the macro. */
#define DEFINE_PARETO(NAME, T)                                                                           \
    void NAME(const T* pts, int N, int D, int remove_duplicates, uint8_t* keep) {                        \
        for (int i = 0; i < N; ++i) {                                                                    \
            const T* xi = pts + (size_t)i * D;                                                           \
            long long n_ge = 0, mult = 0;                                                                \
            int any_not_greater = 0, first = 1;                                                          \
            for (int j = 0; j < N; ++j) {                                                                \
                const T* xj = pts + (size_t)j * D;                                                       \
                int ge = 1, gt = 1, eq = 1;                                                              \
                for (int r = 0; r < D; ++r) {                                                            \
                    ge = ge && (xi[r] <= xj[r]);                                                         \
                    gt = gt && (xi[r] < xj[r]);                                                          \
                    eq = eq && (xi[r] == xj[r]);                                                         \
                }                                                                                        \
                n_ge += ge;                                                                              \
                mult += eq;                                                                              \
                if (!gt) any_not_greater = 1;                                                            \
                if (eq && j < i) first = 0;                                                              \
            }                                                                                            \
            int c1 = (n_ge == mult) && (mult > 0); /* a NaN row has mult == 0: dropped (Appendix A.5) */ \
            keep[i] = (uint8_t)(c1 && any_not_greater && (!remove_duplicates || first));                 \
        }                                                                                                \
    }
DEFINE_PARETO(oracle_pareto_mask_f32, float)
DEFINE_PARETO(oracle_pareto_mask_f64, double)

/* SumTree.sample, common/prioritized_buffer.py:30-54, with the uniform draws supplied by the caller.
 * levels: concatenated level arrays, root first (level l at offset 2^l - 1). */
void oracle_sumtree_sample(const double* levels, int n_levels, const double* query, int B, int64_t* idx) {
    for (int b = 0; b < B; ++b) {
        double q = query[b];
        int64_t node = 0;
        for (int l = 1; l < n_levels; ++l) {
            node *= 2;
            double left = levels[(((int64_t)1) << l) - 1 + node];
            int greater = q > left;
            node += greater;
            q -= left * (double)greater;
        }
        idx[b] = node;
    }
}

static int cmp_pair(const void* a, const void* b) {
    const int64_t* x = (const int64_t*)a;
    const int64_t* y = (const int64_t*)b;
    if (x[0] != y[0]) return x[0] < y[0] ? -1 : 1;
    return x[1] < y[1] ? -1 : (x[1] > y[1]);
}

/* SumTree.batch_set, common/prioritized_buffer.py:69-82: np.unique(idx, return_index) -> sorted unique leaves with the
 * FIRST occurrence's priority; diff = new - old; np.add.at per level in sorted order; node_index //= 2 */
void oracle_sumtree_batch_set(double* levels, int n_levels, const int64_t* idx, const double* prio, int B) {
    int64_t* pairs = (int64_t*)malloc(sizeof(int64_t) * 2 * (size_t)B);
    for (int b = 0; b < B; ++b) {
        pairs[2 * b] = idx[b];
        pairs[2 * b + 1] = b;
    }
    qsort(pairs, (size_t)B, 2 * sizeof(int64_t), cmp_pair);
    int m = 0;
    int64_t* uidx = (int64_t*)malloc(sizeof(int64_t) * (size_t)B);
    double* diff = (double*)malloc(sizeof(double) * (size_t)B);
    int64_t leaf_off = (((int64_t)1) << (n_levels - 1)) - 1;
    for (int b = 0; b < B; ++b) {
        if (b == 0 || pairs[2 * b] != pairs[2 * (b - 1)]) {
            uidx[m] = pairs[2 * b];
            diff[m] = prio[pairs[2 * b + 1]] - levels[leaf_off + pairs[2 * b]];
            ++m;
        }
    }
    for (int l = n_levels - 1; l >= 0; --l) {
        int64_t off = (((int64_t)1) << l) - 1;
        for (int u = 0; u < m; ++u) {
            levels[off + uidx[u]] += diff[u];
            uidx[u] /= 2;
        }
    }
    free(pairs);
    free(uidx);
    free(diff);
}

/* polyak_update, common/networks.py:121-139: copy_ if tau == 1 else mul_(1 - tau) then th.add(alpha=tau) (ATen fmadd) */
void oracle_polyak(const float* param, float* target, int64_t n, double tau) {
    if (tau == 1.0) {
        memcpy(target, param, sizeof(float) * (size_t)n);
        return;
    }
    float omt = (float)(1.0 - tau), tf = (float)tau;
    for (int64_t e = 0; e < n; ++e) {
        float m = target[e] * omt;
        target[e] = fmaf(tf, param[e], m);
    }
}
