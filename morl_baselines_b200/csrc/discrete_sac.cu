// discrete_sac.cu -- discrete-action MOSAC (reference single_policy/ser/mosac_discrete_action.py:445-530).
//
// morl_discrete_sac_target_f32     : the soft target, an expectation under the actor's softmax over all actions (:452-464)
// morl_discrete_sac_actor_loss_f32 : actor loss, its closed-form gradient w.r.t. the logits, and the temperature loss (:478-498)
//
// One thread owns one row; actions are walked in ascending order.  exp and log are the two portable routines below, written
// with IEEE-rounded intrinsics only, so tests/discrete_sac_oracle.c restates them operation for operation and the kernels equal it
// bit for bit.  The loss reductions are deterministic: fixed-shape block partials (float) + one final sum in double.
#include "common.cuh"

namespace morl {

constexpr int kDsThreads = 256;
constexpr int kDsMaxA = 256;

// e^x: Cody-Waite reduction by ln2, degree-7 Taylor polynomial, scaling by 2^j in two normal-range steps.  Max error 2 ulp
// over the range the kernels use (x <= 0), checked against float64 in tests/test_discrete_sac_oracle_cpu.py.
__device__ __forceinline__ float ds_exp(float x) {
    if (x != x) return x;
    if (x < -104.0f) return 0.0f;
    if (x > 89.0f) return __int_as_float(0x7f800000);
    const float j = rintf(__fmul_rn(x, 1.44269502f));
    float r = __fmaf_rn(j, -0.693145751953125f, x);
    r = __fmaf_rn(j, -1.42860677e-06f, r);
    float p = 1.98412698e-04f;
    p = __fmaf_rn(p, r, 1.38888889e-03f);
    p = __fmaf_rn(p, r, 8.33333333e-03f);
    p = __fmaf_rn(p, r, 4.16666667e-02f);
    p = __fmaf_rn(p, r, 1.66666667e-01f);
    p = __fmaf_rn(p, r, 0.5f);
    p = __fmaf_rn(p, r, 1.0f);
    p = __fmaf_rn(p, r, 1.0f);
    const int ji = (int)j;
    const int e1 = ji / 2, e2 = ji - e1;
    return __fmul_rn(__fmul_rn(p, __int_as_float((e1 + 127) << 23)), __int_as_float((e2 + 127) << 23));
}

// log x: x = m 2^e with m in [sqrt(1/2), sqrt(2)], log m = 2 atanh(f / (f + 2)) by its odd series to u^9.
__device__ __forceinline__ float ds_log(float x) {
    if (x != x) return x;
    if (x < 0.0f) return __int_as_float(0x7fffffff);
    if (x == 0.0f) return __int_as_float(0xff800000);
    if (x == __int_as_float(0x7f800000)) return x;
    int e = 0;
    if (x < 1.17549435e-38f) {
        x = __fmul_rn(x, 8388608.0f);
        e = -23;
    }
    const int bits = __float_as_int(x);
    e += ((bits >> 23) & 255) - 127;
    float m = __int_as_float((bits & 0x007fffff) | 0x3f800000);
    if (m > 1.41421356f) {
        m = __fmul_rn(m, 0.5f);
        e += 1;
    }
    const float f = __fsub_rn(m, 1.0f);
    const float u = __fdiv_rn(f, __fadd_rn(f, 2.0f));
    const float u2 = __fmul_rn(u, u);
    float q = __fmaf_rn(u2, 0.111111111f, 0.142857143f);
    q = __fmaf_rn(q, u2, 0.2f);
    q = __fmaf_rn(q, u2, 0.333333333f);
    const float h = __fadd_rn(u, u);
    const float lm = __fmaf_rn(__fmul_rn(h, u2), q, h);
    const float ef = (float)e;
    return __fmaf_rn(ef, 0.693145751953125f, __fmaf_rn(ef, 1.42860677e-06f, lm));
}

// th.min(a, b): NaN if either operand is NaN (not fminf)
__device__ __forceinline__ float nan_min(float a, float b) {
    if (a != a || b != b) return __int_as_float(0x7fffffff);
    return a < b ? a : b;
}

// max (NaN-propagating, as th.max / log_softmax), sum of e^(x - max) in action order, log of that sum
struct SoftmaxRow {
    float mx, s, lse;
};

__device__ __forceinline__ SoftmaxRow softmax_row(const float* __restrict__ x, int A) {
    SoftmaxRow r;
    r.mx = __ldg(x);
    for (int a = 1; a < A; ++a) {
        const float v = __ldg(x + a);
        if (v > r.mx || v != v) r.mx = v;
    }
    r.s = 0.f;
    for (int a = 0; a < A; ++a) r.s = __fadd_rn(r.s, ds_exp(__fsub_rn(__ldg(x + a), r.mx)));
    r.lse = ds_log(r.s);
    return r;
}

// m[a] = min_n w . q_n[k, a, :]
template <int D>
__device__ __forceinline__ float critic_min(const float* __restrict__ q_nets, int n_nets, size_t net_stride, size_t off, const float (&wv)[D]) {
    float m = 0.f;
    for (int n = 0; n < n_nets; ++n) {
        float q[D];
#pragma unroll
        for (int r = 0; r < D; ++r) q[r] = __ldg(q_nets + n * net_stride + off + r);
        const float s = dotw<D, MORL_DOT_UNFUSED>(wv, q);
        m = (n == 0) ? s : nan_min(m, s);
    }
    return m;
}

template <int D>
__global__ void __launch_bounds__(kDsThreads) discrete_sac_target_kernel(const float* __restrict__ q_nets, int n_nets, const float* __restrict__ logits,
                                                                         const float* __restrict__ w, int w_rows, int w_map,
                                                                         const float* __restrict__ reward, const float* __restrict__ done,
                                                                         const float* __restrict__ alpha_dev, float gamma, int N, int A,
                                                                         float* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= N) return;
    const float alpha = __ldg(alpha_dev);
    float wv[D];
    const int wi = map_row(k, w_rows, N, w_map);
#pragma unroll
    for (int r = 0; r < D; ++r) wv[r] = __ldg(w + (size_t)wi * D + r);
    const float* x = logits + (size_t)k * A;
    const SoftmaxRow sm = softmax_row(x, A);
    const size_t net_stride = (size_t)N * A * D;
    float v = 0.f;
    for (int a = 0; a < A; ++a) {
        const float z = __fsub_rn(__ldg(x + a), sm.mx);
        const float lp = __fsub_rn(z, sm.lse);
        if (lp == __int_as_float(0xff800000)) continue;  // -inf logit: p = 0, the action leaves the expectation
        const float p = __fdiv_rn(ds_exp(z), sm.s);
        const float m = critic_min<D>(q_nets, n_nets, net_stride, ((size_t)k * A + a) * D, wv);
        v = __fadd_rn(v, __fmul_rn(p, __fsub_rn(m, __fmul_rn(alpha, lp))));
    }
    float rv[D];
#pragma unroll
    for (int r = 0; r < D; ++r) rv[r] = __ldg(reward + (size_t)k * D + r);
    out[k] = bellman(dotw<D, MORL_DOT_UNFUSED>(wv, rv), __ldg(done + k), gamma, v);
}

__device__ __forceinline__ float ds_block_sum(float v, float* red) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (warp == 0) {
        t = (lane < (blockDim.x >> 5)) ? red[lane] : 0.f;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
    }
    return t;  // valid in thread 0
}

template <int D>
__global__ void __launch_bounds__(kDsThreads) discrete_sac_actor_kernel(const float* __restrict__ logits, const float* __restrict__ q_nets, int n_nets,
                                                                        const float* __restrict__ w, int w_rows, int w_map,
                                                                        const float* __restrict__ alpha_dev, const float* __restrict__ log_alpha,
                                                                        float target_entropy, int N, int A, float inv_na,
                                                                        float* __restrict__ dlogits, float* __restrict__ partials) {
    __shared__ float red[kDsThreads / 32];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    float l = 0.f, al = 0.f, c = 0.f;
    if (k < N) {
        const float alpha = __ldg(alpha_dev);
        const float t = log_alpha ? -ds_exp(__ldg(log_alpha)) : 0.f;
        float wv[D];
        const int wi = map_row(k, w_rows, N, w_map);
#pragma unroll
        for (int r = 0; r < D; ++r) wv[r] = __ldg(w + (size_t)wi * D + r);
        const float* x = logits + (size_t)k * A;
        float* g = dlogits ? dlogits + (size_t)k * A : nullptr;
        const SoftmaxRow sm = softmax_row(x, A);
        const size_t net_stride = (size_t)N * A * D;
        for (int a = 0; a < A; ++a) {
            const float z = __fsub_rn(__ldg(x + a), sm.mx);
            const float lp = __fsub_rn(z, sm.lse);
            if (lp == __int_as_float(0xff800000)) continue;
            const float p = __fdiv_rn(ds_exp(z), sm.s);
            const float m = critic_min<D>(q_nets, n_nets, net_stride, ((size_t)k * A + a) * D, wv);
            const float f = __fsub_rn(__fmul_rn(alpha, lp), m);
            l = __fadd_rn(l, __fmul_rn(p, f));
            if (log_alpha) {
                const float u = __fadd_rn(lp, target_entropy);
                c = __fadd_rn(c, __fmul_rn(p, u));
                al = __fadd_rn(al, __fmul_rn(p, __fmul_rn(t, u)));
            }
            if (g) g[a] = f;  // f parked in the output row until the row's sum l is known
        }
        if (g) {
            for (int a = 0; a < A; ++a) {
                const float z = __fsub_rn(__ldg(x + a), sm.mx);
                const float lp = __fsub_rn(z, sm.lse);
                float v = 0.f;
                if (lp != __int_as_float(0xff800000)) {
                    const float p = __fdiv_rn(ds_exp(z), sm.s);
                    v = __fmul_rn(__fmul_rn(p, __fsub_rn(g[a], l)), inv_na);
                }
                g[a] = v;
            }
        }
    }
    const float s0 = ds_block_sum(l, red);
    const float s1 = ds_block_sum(al, red);
    const float s2 = ds_block_sum(c, red);
    if (threadIdx.x == 0) {
        partials[3 * blockIdx.x + 0] = s0;
        partials[3 * blockIdx.x + 1] = s1;
        partials[3 * blockIdx.x + 2] = s2;
    }
}

__global__ void __launch_bounds__(kDsThreads) discrete_sac_finalize_kernel(const float* __restrict__ partials, int n_blocks, double inv_na,
                                                                           const float* __restrict__ log_alpha, float* __restrict__ actor_loss,
                                                                           float* __restrict__ alpha_loss, float* __restrict__ dlog_alpha) {
    __shared__ double red[3][kDsThreads];
    double s[3] = {0.0, 0.0, 0.0};
    for (int b = threadIdx.x; b < n_blocks; b += blockDim.x)
#pragma unroll
        for (int i = 0; i < 3; ++i) s[i] += (double)partials[3 * b + i];
#pragma unroll
    for (int i = 0; i < 3; ++i) red[i][threadIdx.x] = s[i];
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h)
#pragma unroll
            for (int i = 0; i < 3; ++i) red[i][threadIdx.x] += red[i][threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        actor_loss[0] = (float)(red[0][0] * inv_na);
        if (log_alpha) {
            const float t = -ds_exp(__ldg(log_alpha));
            alpha_loss[0] = (float)(red[1][0] * inv_na);
            dlog_alpha[0] = (float)((double)t * red[2][0] * inv_na);
        }
    }
}

static int check_ds(const char* fn, int n_nets, int N, int A, int D, int w_rows, int w_map) {
    MORL_REQUIRE(n_nets > 0 && N > 0 && A > 0 && D > 0, MORL_ERR_SHAPE, "%s: bad shape n_nets=%d N=%d A=%d D=%d", fn, n_nets, N, A, D);
    MORL_REQUIRE(A <= kDsMaxA, MORL_ERR_UNSUPPORTED, "%s: A=%d > %d", fn, A, kDsMaxA);
    MORL_REQUIRE(D <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "%s: D=%d > %d", fn, D, MORL_MAX_D);
    MORL_REQUIRE(w_map == MORL_MAP_TILE || w_map == MORL_MAP_BLOCK, MORL_ERR_UNSUPPORTED, "%s: bad w_map %d", fn, w_map);
    MORL_REQUIRE(w_rows > 0 && w_rows <= N && N % w_rows == 0, MORL_ERR_SHAPE, "%s: w_rows=%d must divide N=%d", fn, w_rows, N);
    return MORL_OK;
}

}  // namespace morl

extern "C" int morl_discrete_sac_target_f32(const float* q_nets, int n_nets, const float* logits, const float* w, int w_rows, int w_map,
                                            const float* reward, const float* done, const float* alpha, float gamma, int N, int A, int D,
                                            float* target_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(q_nets && logits && w && reward && done && alpha && target_out, MORL_ERR_NULL,
                 "morl_discrete_sac_target_f32: NULL pointer argument");
    int rc = check_ds("morl_discrete_sac_target_f32", n_nets, N, A, D, w_rows, w_map);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int blocks = (N + kDsThreads - 1) / kDsThreads;
    MORL_DISPATCH_D(D, (discrete_sac_target_kernel<kD><<<blocks, kDsThreads, 0, st>>>(q_nets, n_nets, logits, w, w_rows, w_map, reward, done,
                                                                                      alpha, gamma, N, A, target_out)));
    return check_launch("morl_discrete_sac_target_f32");
}

extern "C" size_t morl_discrete_sac_workspace_bytes(int n_rows) {
    if (n_rows <= 0) return 0;
    const size_t blocks = ((size_t)n_rows + morl::kDsThreads - 1) / morl::kDsThreads;
    return blocks * 3 * sizeof(float);
}

extern "C" int morl_discrete_sac_actor_loss_f32(const float* logits, const float* q_nets, int n_nets, const float* w, int w_rows, int w_map,
                                                const float* alpha, const float* log_alpha, float target_entropy, int N, int A, int D,
                                                float* actor_loss_out, float* dlogits, float* alpha_loss_out, float* dlog_alpha_out,
                                                void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(logits && q_nets && w && alpha && actor_loss_out && workspace, MORL_ERR_NULL,
                 "morl_discrete_sac_actor_loss_f32: NULL pointer argument");
    MORL_REQUIRE(!log_alpha || (alpha_loss_out && dlog_alpha_out), MORL_ERR_NULL,
                 "morl_discrete_sac_actor_loss_f32: log_alpha given without alpha_loss_out / dlog_alpha_out");
    int rc = check_ds("morl_discrete_sac_actor_loss_f32", n_nets, N, A, D, w_rows, w_map);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int blocks = (N + kDsThreads - 1) / kDsThreads;
    const double inv_na = 1.0 / ((double)N * A);
    float* partials = static_cast<float*>(workspace);
    MORL_DISPATCH_D(D, (discrete_sac_actor_kernel<kD><<<blocks, kDsThreads, 0, st>>>(logits, q_nets, n_nets, w, w_rows, w_map, alpha, log_alpha,
                                                                                     target_entropy, N, A, (float)inv_na, dlogits, partials)));
    rc = check_launch("morl_discrete_sac_actor_loss_f32");
    if (rc) return rc;
    discrete_sac_finalize_kernel<<<1, kDsThreads, 0, st>>>(partials, blocks, inv_na, log_alpha, actor_loss_out, alpha_loss_out, dlog_alpha_out);
    return check_launch("morl_discrete_sac_actor_loss_f32(finalize)");
}
