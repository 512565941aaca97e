// moq.cu -- multi-policy scalarised Q-learning's tables on the device: batched greedy / GPI actions, and one environment step of one policy
// with its Dyna-Q model updates.
//
// Replaces the per-step host work of the reference's MOQLearning (single_policy/ser/mo_q_learning.py:137-208), its TabularModel
// (common/model_based/tabular_model.py:29-49, 91-122) and MPMOQLearning's _gpi_action / max_scalar_q_value (mp_mo_q_learning.py:125-143).
// Layout (caller-owned, nothing allocated here): q f64 [S, P, A, d] (state-major, so one state's GPI read is one span), visited u8 [S, P],
// pairs int32 [M, 3] (s, a, number of outcomes), outcomes int32 [M, K, 2] (next state, terminal), counts int64 [M, K], out_reward
// f64 [M, K, d], tree f64 [2^18 - 1] (the reference's SumTree(1e5)), status int32 [2].
//
// Rounding: every operation is one IEEE float64 operation in numpy's order, spelled with the _rn intrinsics so no FMA contraction can
// change a bit.  w . v adds the products left to right.  The random draws come from the host, by value.
#include "sumtree.cuh"

namespace morl {

constexpr int kMoqThreads = 256;
constexpr int kMoqWarps = kMoqThreads / 32;
constexpr int kMoqMaxA = 64;
constexpr int kMoqMaxDyna = 64;  // Dyna updates per launch: longer loops are consecutive launches
constexpr int kMoqActRows = 32;  // rows per act launch
constexpr int kMoqLevels = 18;   // SumTree(max_size=1e5): ceil(log2(1e5)) + 1 levels
constexpr int kMoqReal = 8;      // launch flag: this launch runs the real transition before its Dyna updates

struct MoqVec {
    double v[MORL_MAX_D];
};

struct MoqActRows {
    int state[kMoqActRows];
    int policy[kMoqActRows];
    double w[kMoqActRows][MORL_MAX_D];
};

struct MoqDyna {
    int pick[kMoqMaxDyna];       // uniform pair index (random.randint)
    double u[kMoqMaxDyna];       // prioritised walk: query = root * u
    double choice[kMoqMaxDyna];  // random.random() of random.choices
};

struct MoqReal {
    int s, a, s_next, terminal, pair, outcome;
};

struct MoqTable {
    double* q;
    unsigned char* visited;
    int P, A, d;
};

__device__ __forceinline__ double moq_dot(const double* v, const double* w, int d) {
    double acc = __dmul_rn(v[0], w[0]);
    for (int c = 1; c < d; ++c) acc = __dadd_rn(acc, __dmul_rn(v[c], w[c]));
    return acc;
}

// numpy's argmax order: the first NaN, else the first maximum
__device__ __forceinline__ bool moq_better(double v, int i, double bv, int bi) {
    const bool vn = isnan(v), bn = isnan(bv);
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// Greedy entry of `state` under weights w (shared): policy p's actions (p >= 0) or every (policy, action) of the first n_pol policies in
// row-major order (p < 0).  A state the policy never visited (or state -1) scores 0.  Every thread returns the winner's value and flat index.
__device__ void moq_greedy(const MoqTable& t, int state, int p, int n_pol, const double* w, double* rv, int* ri, double& best_v, int& best_i) {
    const int n = p < 0 ? n_pol * t.A : t.A;
    double v = -INFINITY;
    int bi = 0x7fffffff;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        const int pp = p < 0 ? k / t.A : p, a = p < 0 ? k - pp * t.A : k;
        double x = 0.0;
        if (state >= 0 && t.visited[(size_t)state * t.P + pp]) x = moq_dot(t.q + (((size_t)state * t.P + pp) * t.A + a) * t.d, w, t.d);
        if (moq_better(x, k, v, bi)) {
            v = x;
            bi = k;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (moq_better(ov, oi, v, bi)) {
            v = ov;
            bi = oi;
        }
    }
    if ((threadIdx.x & 31) == 0) {
        rv[threadIdx.x >> 5] = v;
        ri[threadIdx.x >> 5] = bi;
    }
    __syncthreads();
    v = rv[0];
    bi = ri[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
        if (moq_better(rv[k], ri[k], v, bi)) {
            v = rv[k];
            bi = ri[k];
        }
    __syncthreads();  // rv / ri free again
    best_v = v;
    best_i = bi;
}

// One row per block: its greedy action, whether the policy has visited the state (own-policy rows; 0 for GPI rows) and the best value.
__global__ void __launch_bounds__(kMoqThreads) moq_act_kernel(MoqTable t, int n_pol, const __grid_constant__ MoqActRows rows, int* __restrict__ out,
                                                              double* __restrict__ value) {
    __shared__ double w[MORL_MAX_D];
    __shared__ double rv[kMoqWarps];
    __shared__ int ri[kMoqWarps];
    const int row = blockIdx.x, s = rows.state[row], p = rows.policy[row];
    if (threadIdx.x < t.d) w[threadIdx.x] = rows.w[row][threadIdx.x];
    __syncthreads();
    double v;
    int k;
    moq_greedy(t, s, p, n_pol, w, rv, ri, v, k);
    if (threadIdx.x == 0) {
        out[2 * row] = k % t.A;
        out[2 * row + 1] = (p >= 0 && s >= 0 && t.visited[(size_t)s * t.P + p]) ? 1 : 0;
        if (value) value[row] = v;
    }
}

struct MoqStepSmem {
    double w[MORL_MAX_D];
    double r[MORL_MAX_D];
    double rv[kMoqWarps];
    int ri[kMoqWarps];
    int s, a, s2, term, pair, stop;
    double prio;
};

// One TD update of policy p on (s, a, r, s2, term) held in shared memory (mo_q_learning.py:177-184 / 199-205), then, with priorities, the
// GPI-PD priority (:144-157) set at leaf `pair` of the tree.
__device__ void moq_td(const MoqTable& t, MoqStepSmem& sm, int p, int n_pol, bool gpi, bool prioritize, double gamma, double lr, double min_p,
                       double alpha, double* tree) {
    const int s = sm.s, a = sm.a, s2 = sm.s2;
    if (threadIdx.x == 0) {
        t.visited[(size_t)s * t.P + p] = 1;
        t.visited[(size_t)s2 * t.P + p] = 1;
    }
    __syncthreads();
    double best;
    int k;
    moq_greedy(t, s2, gpi ? -1 : p, n_pol, sm.w, sm.rv, sm.ri, best, k);
    const double cg = __dmul_rn((double)(1 - sm.term), gamma);  // (1 - terminal) * gamma
    if (threadIdx.x < t.d) {
        const int c = threadIdx.x;
        double* qsa = t.q + (((size_t)s * t.P + p) * t.A + a) * t.d;
        const double mq = t.q[(((size_t)s2 * t.P + p) * t.A + k % t.A) * t.d + c];
        const double td = __dsub_rn(__dadd_rn(sm.r[c], __dmul_rn(cg, mq)), qsa[c]);
        qsa[c] = __dadd_rn(qsa[c], __dmul_rn(lr, td));
    }
    __syncthreads();
    if (!prioritize) return;
    // max_scalar_q_value(s2, w) over every policy: the GPI scan's maximum, unless this update changed a value of s2
    if (!gpi || s == s2) moq_greedy(t, s2, -1, n_pol, sm.w, sm.rv, sm.ri, best, k);
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) {
            const double dr = moq_dot(sm.r, sm.w, t.d);
            const double dq = moq_dot(t.q + (((size_t)s * t.P + p) * t.A + a) * t.d, sm.w, t.d);
            const double x = fabs(__dsub_rn(__dadd_rn(dr, __dmul_rn(cg, best)), dq));
            sm.prio = pow(min_p > x ? min_p : x, alpha);  // max(|priority|, min_priority) ** alpha
        }
        __syncwarp();
        st_set_warp(tree, kMoqLevels, sm.pair, sm.prio);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kMoqThreads) moq_step_kernel(MoqTable t, int* __restrict__ pairs, int* __restrict__ outcomes,
                                                               long long* __restrict__ counts, double* __restrict__ out_reward, double* tree,
                                                               int* __restrict__ status, int K, int n_pol, int p, int flags, double gamma, double lr,
                                                               double min_p, double alpha, const __grid_constant__ MoqVec wv,
                                                               const __grid_constant__ MoqVec rv, MoqReal real, int n_pairs,
                                                               int n_updates, const __grid_constant__ MoqDyna dyna) {
    __shared__ MoqStepSmem sm;
    if (status[0] != 0) return;  // an earlier launch failed: leave everything as it is for the report
    const bool gpi = flags & MORL_MOQ_GPI, model = flags & MORL_MOQ_MODEL, prioritize = flags & MORL_MOQ_PRIORITIZE;
    if (threadIdx.x < t.d) {
        sm.w[threadIdx.x] = wv.v[threadIdx.x];
        sm.r[threadIdx.x] = rv.v[threadIdx.x];
    }
    if (threadIdx.x == 0) {
        sm.s = real.s;
        sm.a = real.a;
        sm.s2 = real.s_next;
        sm.term = real.terminal;
        sm.pair = real.pair;
    }
    __syncthreads();
    if (flags & kMoqReal) {
        moq_td(t, sm, p, n_pol, gpi, prioritize, gamma, lr, min_p, alpha, tree);
        if (model && threadIdx.x == 0) {  // TabularModel.update (tabular_model.py:29-49); the tree leaf was set by moq_td
            const int m = real.pair, o = real.outcome;
            pairs[3 * m] = real.s;
            pairs[3 * m + 1] = real.a;
            pairs[3 * m + 2] = max(pairs[3 * m + 2], o + 1);
            outcomes[2 * ((size_t)m * K + o)] = real.s_next;
            outcomes[2 * ((size_t)m * K + o) + 1] = real.terminal;
            for (int c = 0; c < t.d; ++c) out_reward[((size_t)m * K + o) * t.d + c] = sm.r[c];
            counts[(size_t)m * K + o] += 1;
        }
    }
    for (int j = 0; j < n_updates; ++j) {
        __syncthreads();
        if (threadIdx.x == 0) {  // TabularModel.random_transition (:91-113)
            long long m;
            sm.stop = 0;
            if (prioritize) {
                m = st_walk(tree, kMoqLevels, __dmul_rn(tree[0], dyna.u[j]));
                if (m >= n_pairs) {  // the reference's IndexError
                    status[0] = 1;
                    status[1] = (int)m;
                    sm.stop = 1;
                }
            } else {
                m = dyna.pick[j];
            }
            if (!sm.stop) {
                // random.choices(outcomes, weights=counts / counts.sum()): itertools.accumulate, then bisect_right(cum, random() * total, 0, n - 1)
                const int n = pairs[3 * m + 2];
                const long long* cnt = counts + (size_t)m * K;
                long long tot = 0;
                for (int o = 0; o < n; ++o) tot += cnt[o];
                const double ft = (double)tot;
                double total = 0.0;
                for (int o = 0; o < n; ++o) total = o == 0 ? __ddiv_rn((double)cnt[0], ft) : __dadd_rn(total, __ddiv_rn((double)cnt[o], ft));
                const double x = __dmul_rn(dyna.choice[j], __dadd_rn(total, 0.0));
                int o = 0;
                double cum = __ddiv_rn((double)cnt[0], ft);
                while (o < n - 1 && !(x < cum)) cum = __dadd_rn(cum, __ddiv_rn((double)cnt[++o], ft));
                sm.s = pairs[3 * m];
                sm.a = pairs[3 * m + 1];
                sm.s2 = outcomes[2 * ((size_t)m * K + o)];
                sm.term = outcomes[2 * ((size_t)m * K + o) + 1];
                sm.pair = (int)m;
                for (int c = 0; c < t.d; ++c) sm.r[c] = out_reward[((size_t)m * K + o) * t.d + c];
            }
        }
        __syncthreads();
        if (sm.stop) return;
        moq_td(t, sm, p, n_pol, gpi, prioritize, gamma, lr, min_p, alpha, tree);
    }
}

static MoqVec moq_vec(const double* p, int d) {
    MoqVec v = {};
    for (int c = 0; c < d; ++c) v.v[c] = p[c];
    return v;
}

}  // namespace morl

extern "C" int morl_moq_supported(int n_actions, int d) {
    return n_actions >= 1 && n_actions <= morl::kMoqMaxA && d >= 1 && d <= MORL_MAX_D ? 1 : 0;
}

extern "C" int morl_moq_act_f64(const double* q, const unsigned char* visited, int S, int P, int A, int d, int n_policies, const int* state,
                                const int* policy, const double* w, int n, int* out, double* value, void* stream) {
    using namespace morl;
    MORL_REQUIRE(q && visited && state && policy && w && out, MORL_ERR_NULL, "morl_moq_act_f64: NULL pointer argument");
    MORL_REQUIRE(morl_moq_supported(A, d), MORL_ERR_UNSUPPORTED, "morl_moq_act_f64: supports 1 <= A <= %d, 1 <= d <= %d (got A=%d, d=%d)",
                 kMoqMaxA, MORL_MAX_D, A, d);
    MORL_REQUIRE(S >= 1 && P >= 1 && n_policies >= 1 && n_policies <= P && n >= 0, MORL_ERR_SHAPE,
                 "morl_moq_act_f64: bad shape S=%d P=%d n_policies=%d n=%d", S, P, n_policies, n);
    for (int i = 0; i < n; ++i)
        MORL_REQUIRE(state[i] >= -1 && state[i] < S && policy[i] >= -1 && policy[i] < n_policies, MORL_ERR_SHAPE,
                     "morl_moq_act_f64: row %d: state=%d outside [-1, %d) or policy=%d outside [-1, %d)", i, state[i], S, policy[i], n_policies);
    const MoqTable t = {const_cast<double*>(q), const_cast<unsigned char*>(visited), P, A, d};
    for (int r0 = 0; r0 < n; r0 += kMoqActRows) {
        const int m = min(kMoqActRows, n - r0);
        MoqActRows rows = {};
        for (int i = 0; i < m; ++i) {
            rows.state[i] = state[r0 + i];
            rows.policy[i] = policy[r0 + i];
            for (int c = 0; c < d; ++c) rows.w[i][c] = w[(size_t)(r0 + i) * d + c];
        }
        moq_act_kernel<<<m, kMoqThreads, 0, static_cast<cudaStream_t>(stream)>>>(t, n_policies, rows, out + 2 * r0, value ? value + r0 : nullptr);
        const int rc = check_launch("morl_moq_act_f64");
        if (rc != MORL_OK) return rc;
    }
    return MORL_OK;
}

extern "C" int morl_moq_step_f64(double* q, unsigned char* visited, int* pairs, int* outcomes, long long* counts, double* out_reward, double* tree,
                                 int* status, int S, int P, int A, int d, int M, int K, int n_policies, int p, int s, int a, int s_next, int terminal,
                                 int pair, int outcome, int n_pairs, const double* w, const double* reward, int flags, double gamma, double lr,
                                 double min_priority, double alpha, int n_updates, const int* pick, const double* u, const double* choice,
                                 void* stream) {
    using namespace morl;
    const bool model = flags & MORL_MOQ_MODEL, prioritize = flags & MORL_MOQ_PRIORITIZE;
    MORL_REQUIRE(q && visited && status && w && reward && (!model || (pairs && outcomes && counts && out_reward)) && (!prioritize || tree) &&
                     (!model || n_updates == 0 || (choice && (prioritize ? u != nullptr : pick != nullptr))),
                 MORL_ERR_NULL, "morl_moq_step_f64: NULL pointer argument");
    MORL_REQUIRE(morl_moq_supported(A, d), MORL_ERR_UNSUPPORTED, "morl_moq_step_f64: supports 1 <= A <= %d, 1 <= d <= %d (got A=%d, d=%d)",
                 kMoqMaxA, MORL_MAX_D, A, d);
    MORL_REQUIRE((flags & ~(MORL_MOQ_GPI | MORL_MOQ_MODEL | MORL_MOQ_PRIORITIZE)) == 0 && (model || !prioritize), MORL_ERR_SHAPE,
                 "morl_moq_step_f64: bad flags %d", flags);
    MORL_REQUIRE(S >= 1 && P >= 1 && n_policies >= 1 && n_policies <= P && p >= 0 && p < n_policies && s >= 0 && s < S && s_next >= 0 &&
                     s_next < S && a >= 0 && a < A && n_updates >= 0 && (terminal == 0 || terminal == 1),
                 MORL_ERR_SHAPE, "morl_moq_step_f64: bad step S=%d P=%d n_policies=%d p=%d s=%d a=%d s_next=%d terminal=%d n_updates=%d", S, P,
                 n_policies, p, s, a, s_next, terminal, n_updates);
    if (model) {
        MORL_REQUIRE(M >= 1 && K >= 1 && n_pairs >= 1 && n_pairs <= M && n_pairs <= (1 << (kMoqLevels - 1)) && pair >= 0 && pair < n_pairs &&
                         outcome >= 0 && outcome < K,
                     MORL_ERR_SHAPE, "morl_moq_step_f64: bad model shape M=%d K=%d n_pairs=%d pair=%d outcome=%d", M, K, n_pairs, pair, outcome);
        for (int j = 0; j < n_updates && !prioritize; ++j)
            MORL_REQUIRE(pick[j] >= 0 && pick[j] < n_pairs, MORL_ERR_SHAPE, "morl_moq_step_f64: pick[%d]=%d outside [0, %d)", j, pick[j], n_pairs);
    } else {
        n_updates = 0;
    }
    const MoqTable t = {q, visited, P, A, d};
    const MoqReal real = {s, a, s_next, terminal, pair, outcome};
    const MoqVec wv = moq_vec(w, d), rv = moq_vec(reward, d);
    int kflags = flags | kMoqReal;
    int j0 = 0;
    do {
        const int m = min(kMoqMaxDyna, n_updates - j0);
        MoqDyna dy = {};
        for (int j = 0; j < m; ++j) {
            if (pick) dy.pick[j] = pick[j0 + j];
            if (u) dy.u[j] = u[j0 + j];
            dy.choice[j] = choice[j0 + j];
        }
        moq_step_kernel<<<1, kMoqThreads, 0, static_cast<cudaStream_t>(stream)>>>(t, pairs, outcomes, counts, out_reward, tree, status, K,
                                                                                   n_policies, p, kflags, gamma, lr, min_priority, alpha, wv, rv,
                                                                                   real, n_pairs, m, dy);
        const int rc = check_launch("morl_moq_step_f64");
        if (rc != MORL_OK) return rc;
        kflags &= ~kMoqReal;
        j0 += m;
    } while (j0 < n_updates);
    return MORL_OK;
}
