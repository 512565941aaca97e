// eupg.cu -- EUPG's policy network (reference single_policy/esr/eupg.py:22-75) and its episode update (eupg.py:226-270) on CUDA cores.
//
//   x = [obs || accrued reward] [S + d],  a_{l+1} = tanh(W_l a_l + b_l) for the hidden layers,  z = W_L a_L + b_L [A],
//   p = sigmoid(z) / sum_a sigmoid(z_a),  log p_a = log(clamp(p_a, eps, 1 - eps)) with eps = 2^-23 (no gradient where the clamp acts).
//
// The reference also divides sigmoid(z) by its sum over the whole batch before Categorical renormalises every row; that factor cancels
// in p and in its gradient, so it is not computed.
//
// morl_eupg_returns_f32 : discounted forward returns c_t = gamma * c_{t+1} + r_t, backward along T in float32 with the product and the sum
//                         rounded separately, bit-identical to the reference's python loop (eupg.py:263-270)
// morl_eupg_update_f32  : int32 obs -> float, forward, p, clamped log-probability of the taken action, loss = -mean(logp * v), backward.
//                         A FIXED number of CTAs (kEupgCtas) each folds a contiguous range of 16-row tiles, in tile order, into its own
//                         gradient partial; a second launch sums the partials in CTA order into the .grad storages.  The workspace does
//                         not grow with T and the result depends on neither the SM count nor the run.
// morl_eupg_probs_f32   : the forward alone on N rows, writing p (rows and output may be mapped pinned host memory)
//
// Widths are arbitrary in [1, 256] (the reference's default net_arch is [50]); the networks are tiny, so CUDA cores, not tensor cores.
#include "common.cuh"

namespace morl {

constexpr int kEupgThreads = 256;
constexpr int kEupgRows = 16;         // rows per tile
constexpr int kEupgCtas = 128;        // CTAs of the update, whatever T and the card (the reduction order depends on it)
constexpr int kEupgMaxWidth = 256;    // input (S + d) and hidden widths
constexpr int kEupgMaxHidden = 4;
constexpr int kEupgMaxA = 32;
constexpr int kEupgMaxLayers = kEupgMaxHidden + 1;
constexpr int kEupgReturnsSmem = 8192;  // floats of rewards staged in shared memory per step of the returns kernel
constexpr float kEupgEps = 1.1920928955078125e-07f;  // torch.finfo(float32).eps

// The rows a job owns are g, g + groups, ... (rpj of them); unrolled to kEupgRows so the per-row accumulators stay in registers.
#define MORL_EUPG_ROWS(i) _Pragma("unroll") for (int i = 0; i < kEupgRows; ++i) if (i < rpj)

struct EupgShape {
    int L;                       // Linear layers = hidden layers + 1
    int S, d;
    int w[kEupgMaxLayers + 1];   // w[0] = S + d, w[1..L-1] hidden widths, w[L] = A; layer l maps w[l] -> w[l + 1]
    __host__ __device__ int size(int t) const {  // tensor t: 2l = W_l [w[l+1], w[l]], 2l + 1 = b_l [w[l+1]]
        const int l = t >> 1;
        return (t & 1) ? w[l + 1] : w[l + 1] * w[l];
    }
    __host__ __device__ int offset(int t) const {
        int o = 0;
        for (int i = 0; i < t; ++i) o += size(i);
        return o;
    }
    __host__ __device__ int total() const { return offset(2 * L); }
    __host__ __device__ int max_out() const {  // widest layer output (the gradient ping-pong buffers)
        int m = 0;
        for (int l = 1; l <= L; ++l) m = w[l] > m ? w[l] : m;
        return m;
    }
    __host__ __device__ int act_floats() const {  // inputs of every layer, per row
        int s = 0;
        for (int l = 0; l < L; ++l) s += w[l];
        return s;
    }
};

struct EupgParams {
    const float* p[2 * kEupgMaxLayers];
};
struct EupgGrads {
    float* g[2 * kEupgMaxLayers];
};

__host__ __device__ inline size_t eupg_smem_floats(const EupgShape& sh) {
    return (size_t)kEupgRows * (sh.act_floats() + 2 * sh.max_out());
}

// groups of rows per job for a layer with n outputs: the largest power of two <= 256 / n, at most kEupgRows, so that n * groups <= 256 and
// every job runs in one pass of the block
__device__ __forceinline__ int eupg_groups(int n) {
    int g = kEupgThreads / n;
    g = g > kEupgRows ? kEupgRows : g;
    return 1 << (31 - __clz(g));
}

__device__ __forceinline__ float eupg_sigmoid(float z) { return 1.0f / (1.0f + expf(-z)); }

// Shared memory: the inputs of layers 0..L-1, then the two gradient buffers.
__device__ __forceinline__ float* eupg_act(float* base, const EupgShape& sh, int l) {
    int o = 0;
    for (int i = 0; i < l; ++i) o += sh.w[i];
    return base + kEupgRows * o;
}
__device__ __forceinline__ float* eupg_grad_buf(float* base, const EupgShape& sh, int which) {
    return base + kEupgRows * (sh.act_floats() + which * sh.max_out());
}

// out[r, j] = act(b[j] + sum_k W[j, k] in[r, k]) for the tile's rows.  Job (j, g) walks weight row j once and applies it to its rpj rows.
__device__ void eupg_linear(const float* __restrict__ W, const float* __restrict__ b, const float* in, int K, float* out, int N, bool tanh_act) {
    const int groups = eupg_groups(N), rpj = kEupgRows / groups;
    const int job = threadIdx.x;
    if (job < N * groups) {
        const int j = job % N, g = job / N;
        float acc[kEupgRows];
        MORL_EUPG_ROWS(i) acc[i] = 0.f;
        const float* wr = W + (size_t)j * K;
        for (int k = 0; k < K; ++k) {
            const float wv = __ldg(wr + k);
            MORL_EUPG_ROWS(i) acc[i] = fmaf(wv, in[(g + groups * i) * K + k], acc[i]);
        }
        const float bj = __ldg(b + j);
        MORL_EUPG_ROWS(i) {
            const float v = acc[i] + bj;
            out[(g + groups * i) * N + j] = tanh_act ? tanhf(v) : v;
        }
    }
    __syncthreads();
}

// The whole forward of the staged tile: eupg_act(l) holds the inputs of layer l, logits go to `z` [kEupgRows, A].
__device__ void eupg_forward_tile(const EupgParams& P, const EupgShape& sh, float* base, float* z) {
    for (int l = 0; l < sh.L; ++l) {
        const bool last = l == sh.L - 1;
        eupg_linear(P.p[2 * l], P.p[2 * l + 1], eupg_act(base, sh, l), sh.w[l], last ? z : eupg_act(base, sh, l + 1), sh.w[l + 1], !last);
    }
}

__device__ __forceinline__ float eupg_warp_sum(float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// Stages rows [t0, t0 + kEupgRows) of the episode: x = [float(obs) || accrued reward], zero past T.
__device__ __forceinline__ void eupg_stage(float* x, const EupgShape& sh, const int32_t* __restrict__ obs, const float* __restrict__ acc, int ld,
                                           int t0, int T) {
    const int K = sh.w[0], S = sh.S;
    for (int idx = threadIdx.x; idx < kEupgRows * K; idx += kEupgThreads) {
        const int r = idx / K, k = idx % K, row = t0 + r;
        float v = 0.f;
        if (row < T) v = k < S ? __int2float_rn(__ldg(obs + (size_t)row * ld + k)) : __ldg(acc + (size_t)row * ld + (k - S));
        x[idx] = v;
    }
    __syncthreads();
}

// One CTA folds tiles [tile0, tile0 + n_tiles) in order into its partial part[blockIdx.x] (every parameter element) and its loss partial
// (sum of logp * v in double).
__global__ void __launch_bounds__(kEupgThreads) eupg_update_kernel(const __grid_constant__ EupgParams P,
                                                                   const __grid_constant__ EupgShape sh, const int32_t* __restrict__ obs,
                                                                   const float* __restrict__ acc, const int32_t* __restrict__ actions, int ld,
                                                                   const float* __restrict__ v, int v_stride, int T,
                                                                   float* __restrict__ part, double* __restrict__ loss_part) {
    extern __shared__ float smem[];
    __shared__ double red[kEupgThreads / 32];
    float* const D0 = eupg_grad_buf(smem, sh, 0);
    const int L = sh.L, A = sh.w[L];
    const int n_all = (T + kEupgRows - 1) / kEupgRows;
    const int q = n_all / kEupgCtas, rem = n_all % kEupgCtas;
    const int c = blockIdx.x;
    const int first = c * q + min(c, rem), count = q + (c < rem ? 1 : 0);
    const float inv_t = 1.0f / (float)T;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* out = part + (size_t)c * sh.total();
    double lsum = 0.0;

    for (int tile = first; tile < first + count; ++tile) {
        const bool init = tile == first;
        const int t0 = tile * kEupgRows;
        eupg_stage(smem, sh, obs, acc, ld, t0, T);
        eupg_forward_tile(P, sh, smem, D0);

        // p, the clamped log-probability of the taken action, the loss term and dL/dz (one warp per row; A <= 32 so lane a holds z_a):
        //   dL/dz_a = g (1 - sigmoid(z_a)) ([a == action] - p_a),  g = -v / T where the clamp passes the gradient, else 0
        for (int r = warp; r < kEupgRows; r += kEupgThreads / 32) {
            const int row = t0 + r;
            const bool valid = row < T;
            const float z = lane < A ? D0[r * A + lane] : 0.f;
            const float sg = lane < A ? eupg_sigmoid(z) : 0.f;
            const float s = eupg_warp_sum(sg);
            const float p = sg / s;
            const int a = valid ? __ldg(actions + (size_t)row * ld) : 0;
            const float pa = __shfl_sync(0xffffffffu, p, a & 31);
            const float logp = logf(fminf(fmaxf(pa, kEupgEps), 1.0f - kEupgEps));
            const float vt = valid ? __ldg(v + (size_t)row * v_stride) : 0.f;
            if (lane == 0 && valid) lsum += (double)(logp * vt);
            const bool pass = valid && pa >= kEupgEps && pa <= 1.0f - kEupgEps;
            const float g = pass ? -vt * inv_t : 0.f;
            if (lane < A) D0[r * A + lane] = g * (1.0f - sg) * ((lane == a ? 1.0f : 0.0f) - p);
        }
        __syncthreads();

        // backward, last layer first: dz_l is in gradient buffer `cur`; a_l is the input of layer l
        int cur = 0;
        for (int l = L - 1; l >= 0; --l) {
            const int N = sh.w[l + 1], K = sh.w[l];
            const float* dz = eupg_grad_buf(smem, sh, cur);
            const float* a = eupg_act(smem, sh, l);
            float* gw = out + sh.offset(2 * l);
            float* gb = out + sh.offset(2 * l + 1);
            for (int idx = threadIdx.x; idx < N * K; idx += kEupgThreads) {
                const int j = idx / K, k = idx % K;
                float s = 0.f;
#pragma unroll
                for (int r = 0; r < kEupgRows; ++r) s = fmaf(dz[r * N + j], a[r * K + k], s);
                gw[idx] = init ? s : gw[idx] + s;
            }
            for (int j = threadIdx.x; j < N; j += kEupgThreads) {
                float s = 0.f;
#pragma unroll
                for (int r = 0; r < kEupgRows; ++r) s += dz[r * N + j];
                gb[j] = init ? s : gb[j] + s;
            }
            if (l > 0) {
                // dz_{l-1}[r, k] = (sum_j W_l[j, k] dz_l[r, j]) (1 - a_l[r, k]^2)   (a_l = tanh output of layer l - 1)
                const float* W = P.p[2 * l];
                float* nx = eupg_grad_buf(smem, sh, cur ^ 1);
                const int groups = eupg_groups(K), rpj = kEupgRows / groups;
                const int job = threadIdx.x;
                if (job < K * groups) {
                    const int k = job % K, g = job / K;
                    float s[kEupgRows];
                    MORL_EUPG_ROWS(i) s[i] = 0.f;
                    for (int j = 0; j < N; ++j) {
                        const float wv = __ldg(W + (size_t)j * K + k);
                        MORL_EUPG_ROWS(i) s[i] = fmaf(wv, dz[(g + groups * i) * N + j], s[i]);
                    }
                    MORL_EUPG_ROWS(i) {
                        const int r = g + groups * i;
                        const float y = a[r * K + k];
                        nx[r * K + k] = s[i] * (1.0f - y * y);
                    }
                }
            }
            __syncthreads();
            cur ^= 1;
        }
    }

    if (lane == 0) red[warp] = lsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < kEupgThreads / 32; ++i) t += red[i];
        loss_part[c] = t;
    }
}

// Fixed-order sum of the active CTAs' partials into the .grad storages; block 0 also finishes the loss.
__global__ void __launch_bounds__(kEupgThreads) eupg_reduce_kernel(const __grid_constant__ EupgGrads G,
                                                                   const __grid_constant__ EupgShape sh, const float* __restrict__ part,
                                                                   const double* __restrict__ loss_part, int n_parts, int T,
                                                                   float* __restrict__ loss_out) {
    const int total = sh.total();
    int off = 0;
#pragma unroll
    for (int t = 0; t < 2 * kEupgMaxLayers; ++t) {  // unrolled: G.g[t] stays a kernel parameter, not a stack array
        if (t < 2 * sh.L) {
            const int n = sh.size(t);
            for (int q = blockIdx.x * kEupgThreads + threadIdx.x; q < n; q += gridDim.x * kEupgThreads) {
                float s = 0.f;
                for (int c = 0; c < n_parts; ++c) s += __ldg(part + (size_t)c * total + off + q);
                G.g[t][q] = s;
            }
            off += n;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        double l = 0.0;
        for (int c = 0; c < n_parts; ++c) l += loss_part[c];
        loss_out[0] = (float)(-l / (double)T);
    }
}

// Forward alone on N rows x [N, S + d]; out [N, A] = p.  x and out may live in mapped pinned host memory.
__global__ void __launch_bounds__(kEupgThreads) eupg_probs_kernel(const __grid_constant__ EupgParams P,
                                                                  const __grid_constant__ EupgShape sh, const float* x, int N, float* out) {
    extern __shared__ float smem[];
    float* const D0 = eupg_grad_buf(smem, sh, 0);
    const int K = sh.w[0], A = sh.w[sh.L];
    const int r0 = blockIdx.x * kEupgRows;
    const int nr = min(kEupgRows, N - r0);
    for (int idx = threadIdx.x; idx < kEupgRows * K; idx += kEupgThreads) {
        const int r = idx / K;
        smem[idx] = r < nr ? x[(size_t)r0 * K + idx] : 0.f;
    }
    __syncthreads();
    eupg_forward_tile(P, sh, smem, D0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < nr; r += kEupgThreads / 32) {
        const float sg = lane < A ? eupg_sigmoid(D0[r * A + lane]) : 0.f;
        const float s = eupg_warp_sum(sg);
        if (lane < A) out[(size_t)(r0 + r) * A + lane] = sg / s;
    }
}

// c = gamma * c + r_t from t = T - 1 down to 0, per objective, with the product and the sum rounded separately.  CTA b owns objectives
// [256 b, 256 b + dc); its rewards are staged chunk by chunk (last chunk first) in shared memory, one thread per objective runs the
// recurrence, then the chunk is written out.  Objectives are independent, so any number of them is covered.
__global__ void __launch_bounds__(kEupgThreads) eupg_returns_kernel(const float* __restrict__ rewards, int ld, int T, int d, float gamma,
                                                                    float* __restrict__ out) {
    __shared__ float buf[kEupgReturnsSmem];
    const int k0 = blockIdx.x * kEupgThreads, dc = min(kEupgThreads, d - k0);
    const int chunk = kEupgReturnsSmem / dc;
    float c = 0.f;
    for (int hi = T; hi > 0; hi -= chunk) {
        const int lo = max(0, hi - chunk), n = hi - lo;
        for (int idx = threadIdx.x; idx < n * dc; idx += kEupgThreads) {
            const int r = idx / dc, k = idx % dc;
            buf[idx] = __ldg(rewards + (size_t)(lo + r) * ld + k0 + k);
        }
        __syncthreads();
        if (threadIdx.x < dc) {
            const int k = threadIdx.x;
            for (int r = n - 1; r >= 0; --r) {
                c = __fadd_rn(__fmul_rn(gamma, c), buf[r * dc + k]);
                buf[r * dc + k] = c;
            }
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < n * dc; idx += kEupgThreads) {
            const int r = idx / dc, k = idx % dc;
            out[(size_t)(lo + r) * d + k0 + k] = buf[idx];
        }
        __syncthreads();
    }
}

static bool eupg_shape(int obs_dim, int d, const int* hidden, int n_hidden, int n_out, EupgShape* sh) {
    if (obs_dim < 1 || d < 1 || d > MORL_MAX_D || obs_dim + d > kEupgMaxWidth || n_out < 1 || n_out > kEupgMaxA || !hidden || n_hidden < 1 ||
        n_hidden > kEupgMaxHidden)
        return false;
    sh->L = n_hidden + 1;
    sh->S = obs_dim;
    sh->d = d;
    sh->w[0] = obs_dim + d;
    for (int i = 0; i < n_hidden; ++i) {
        if (hidden[i] < 1 || hidden[i] > kEupgMaxWidth) return false;
        sh->w[i + 1] = hidden[i];
    }
    sh->w[sh->L] = n_out;
    for (int l = sh->L + 1; l <= kEupgMaxLayers; ++l) sh->w[l] = 0;
    return true;
}

static size_t eupg_max_smem_bytes() {
    EupgShape m;
    m.L = kEupgMaxLayers;
    m.S = kEupgMaxWidth - 1;
    m.d = 1;
    for (int l = 0; l < kEupgMaxLayers; ++l) m.w[l] = kEupgMaxWidth;
    m.w[kEupgMaxLayers] = kEupgMaxA;
    return eupg_smem_floats(m) * sizeof(float);
}

template <typename T>
static void eupg_tables(const EupgShape& sh, T* const* src, T** dst) {
    for (int t = 0; t < 2 * kEupgMaxLayers; ++t) dst[t] = t < 2 * sh.L ? src[t] : nullptr;
}

}  // namespace morl

extern "C" int morl_eupg_supported(int obs_dim, int d, const int* hidden, int n_hidden, int n_out) {
    morl::EupgShape sh;
    return morl::eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh) ? 1 : 0;
}

extern "C" size_t morl_eupg_workspace_bytes(int obs_dim, int d, const int* hidden, int n_hidden, int n_out) {
    using namespace morl;
    EupgShape sh;
    if (!eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh)) return 0;
    return (size_t)kEupgCtas * sizeof(double) + (size_t)kEupgCtas * (size_t)sh.total() * sizeof(float);
}

extern "C" int morl_eupg_returns_f32(const float* rewards, int ld, int T, int d, float gamma, float* out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(rewards && out, MORL_ERR_NULL, "morl_eupg_returns_f32: NULL pointer argument");
    MORL_REQUIRE(T > 0 && d > 0 && ld >= d, MORL_ERR_SHAPE, "morl_eupg_returns_f32: bad shape T=%d d=%d ld=%d", T, d, ld);
    eupg_returns_kernel<<<(d + kEupgThreads - 1) / kEupgThreads, kEupgThreads, 0, static_cast<cudaStream_t>(stream)>>>(rewards, ld, T, d, gamma, out);
    return check_launch("morl_eupg_returns_f32");
}

extern "C" int morl_eupg_update_f32(const float* const* params, float* const* grads, const int32_t* obs, const float* acc, const int32_t* actions,
                                    int ld, const float* v, int v_stride, int T, int obs_dim, int d, const int* hidden, int n_hidden, int n_out,
                                    float* loss_out, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && grads && obs && acc && actions && v && hidden && loss_out && workspace, MORL_ERR_NULL,
                 "morl_eupg_update_f32: NULL pointer argument");
    MORL_REQUIRE(T > 0 && obs_dim > 0 && d > 0 && n_hidden > 0 && n_out > 0 && v_stride >= 0, MORL_ERR_SHAPE,
                 "morl_eupg_update_f32: bad shape T=%d S=%d d=%d layers=%d A=%d v_stride=%d", T, obs_dim, d, n_hidden, n_out, v_stride);
    EupgShape sh;
    MORL_REQUIRE(eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh), MORL_ERR_UNSUPPORTED,
                 "morl_eupg_update_f32: unsupported configuration S=%d d=%d layers=%d A=%d (morl_eupg_supported)", obs_dim, d, n_hidden, n_out);
    MORL_REQUIRE(ld >= obs_dim + d + 1, MORL_ERR_SHAPE, "morl_eupg_update_f32: ld=%d < S + d + 1", ld);
    EupgParams P;
    EupgGrads G;
    for (int t = 0; t < 2 * sh.L; ++t)
        MORL_REQUIRE(params[t] && grads[t], MORL_ERR_NULL, "morl_eupg_update_f32: NULL parameter or gradient pointer %d", t);
    eupg_tables(sh, params, P.p);
    eupg_tables(sh, grads, G.g);
    const int tiles = (T + kEupgRows - 1) / kEupgRows;
    const int ctas = min(kEupgCtas, tiles);
    double* loss_part = static_cast<double*>(workspace);
    float* part = reinterpret_cast<float*>(loss_part + kEupgCtas);
    set_smem_limit_once<eupg_update_kernel>(eupg_max_smem_bytes());
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    eupg_update_kernel<<<ctas, kEupgThreads, eupg_smem_floats(sh) * sizeof(float), st>>>(P, sh, obs, acc, actions, ld, v, v_stride, T, part,
                                                                                        loss_part);
    const int rblocks = min((sh.total() + kEupgThreads - 1) / kEupgThreads, 4 * sm_count());
    eupg_reduce_kernel<<<rblocks, kEupgThreads, 0, st>>>(G, sh, part, loss_part, ctas, T, loss_out);
    return check_launch("morl_eupg_update_f32");
}

extern "C" int morl_eupg_probs_f32(const float* const* params, const float* x, int N, int obs_dim, int d, const int* hidden, int n_hidden,
                                   int n_out, float* out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && x && hidden && out, MORL_ERR_NULL, "morl_eupg_probs_f32: NULL pointer argument");
    MORL_REQUIRE(N > 0 && obs_dim > 0 && d > 0 && n_hidden > 0 && n_out > 0, MORL_ERR_SHAPE,
                 "morl_eupg_probs_f32: bad shape N=%d S=%d d=%d layers=%d A=%d", N, obs_dim, d, n_hidden, n_out);
    EupgShape sh;
    MORL_REQUIRE(eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh), MORL_ERR_UNSUPPORTED,
                 "morl_eupg_probs_f32: unsupported configuration S=%d d=%d layers=%d A=%d (morl_eupg_supported)", obs_dim, d, n_hidden, n_out);
    EupgParams P;
    for (int t = 0; t < 2 * sh.L; ++t) MORL_REQUIRE(params[t], MORL_ERR_NULL, "morl_eupg_probs_f32: NULL parameter pointer %d", t);
    eupg_tables(sh, params, P.p);
    set_smem_limit_once<eupg_probs_kernel>(eupg_max_smem_bytes());
    eupg_probs_kernel<<<(N + kEupgRows - 1) / kEupgRows, kEupgThreads, eupg_smem_floats(sh) * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
        P, sh, x, N, out);
    return check_launch("morl_eupg_probs_f32");
}
