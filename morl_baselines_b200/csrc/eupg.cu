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
//                         gradient partial; a second launch sums the partials in CTA order into the .grad storages (tile_mlp.cuh).  The workspace does
//                         not grow with T and the result depends on neither the SM count nor the run.
// morl_eupg_probs_f32   : the forward alone on N rows, writing p (rows and output may be mapped pinned host memory)
//
// Widths are arbitrary in [1, 256] (the reference's default net_arch is [50]); the networks are tiny, so CUDA cores, not tensor cores.
#include "tile_mlp.cuh"

namespace morl {

constexpr int kEupgCtas = 128;        // CTAs of the update, whatever T and the card (the reduction order depends on it)
constexpr int kEupgMaxWidth = 256;    // input (S + d) and hidden widths
constexpr int kEupgMaxHidden = 4;
constexpr int kEupgMaxA = 32;
constexpr int kEupgMaxLayers = kEupgMaxHidden + 1;
constexpr int kEupgTensors = 2 * kEupgMaxLayers;
constexpr int kEupgReturnsThreads = 256;  // objectives per CTA of the returns kernel
constexpr int kEupgReturnsSmem = 8192;     // floats of rewards staged in shared memory per step of the returns kernel
constexpr float kEupgEps = 1.1920928955078125e-07f;  // torch.finfo(float32).eps

using EupgParams = ParamTable<kEupgTensors>;
using EupgGrads = GradTable<kEupgTensors>;
using EupgLayout = ParamLayout<kEupgTensors>;

struct EupgShape {
    int L;                       // Linear layers = hidden layers + 1
    int S, d;
    int w[kEupgMaxLayers + 1];   // w[0] = S + d, w[1..L-1] hidden widths, w[L] = A; layer l maps w[l] -> w[l + 1]
    EupgLayout layout() const {  // tensor t: 2l = W_l [w[l+1], w[l]], 2l + 1 = b_l [w[l+1]]
        EupgLayout lay{2 * L, {}};
        for (int l = 0; l < L; ++l) {
            lay.size[2 * l] = w[l + 1] * w[l];
            lay.size[2 * l + 1] = w[l + 1];
        }
        return lay;
    }
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

__host__ __device__ inline size_t eupg_smem_floats(const EupgShape& sh) {
    return (size_t)kTileRows * (sh.act_floats() + 2 * sh.max_out());
}

// Shared memory: the inputs of layers 0..L-1, then the two gradient buffers.
__device__ __forceinline__ float* eupg_act(float* base, const EupgShape& sh, int l) {
    int o = 0;
    for (int i = 0; i < l; ++i) o += sh.w[i];
    return base + kTileRows * o;
}
__device__ __forceinline__ float* eupg_grad_buf(float* base, const EupgShape& sh, int which) {
    return base + kTileRows * (sh.act_floats() + which * sh.max_out());
}

// The whole forward of the staged tile: eupg_act(l) holds the inputs of layer l, logits go to `z` [kTileRows, A].
__device__ void eupg_forward_tile(const EupgParams& P, const EupgShape& sh, float* base, float* z) {
    for (int l = 0; l < sh.L; ++l) {
        const bool last = l == sh.L - 1;
        tile_linear(P.p[2 * l], P.p[2 * l + 1], eupg_act(base, sh, l), sh.w[l], last ? z : eupg_act(base, sh, l + 1), sh.w[l + 1],
                    last ? Act::None : Act::Tanh);
    }
}

// Stages rows [t0, t0 + kTileRows) of the episode: x = [float(obs) || accrued reward], zero past T.
__device__ __forceinline__ void eupg_stage(float* x, const EupgShape& sh, const int32_t* __restrict__ obs, const float* __restrict__ acc, int ld,
                                           int t0, int T) {
    const int K = sh.w[0], S = sh.S;
    for (int idx = threadIdx.x; idx < kTileRows * K; idx += kTileThreads) {
        const int r = idx / K, k = idx % K, row = t0 + r;
        float v = 0.f;
        if (row < T) v = k < S ? __int2float_rn(__ldg(obs + (size_t)row * ld + k)) : __ldg(acc + (size_t)row * ld + (k - S));
        x[idx] = v;
    }
    __syncthreads();
}

// One CTA folds its range of tiles in order into its partial part[blockIdx.x] (every parameter element) and its loss partial (sum of
// logp * v in double).
__global__ void __launch_bounds__(kTileThreads) eupg_update_kernel(const __grid_constant__ EupgParams P, const __grid_constant__ EupgShape sh,
                                                                   const __grid_constant__ EupgLayout lay, const int32_t* __restrict__ obs,
                                                                   const float* __restrict__ acc, const int32_t* __restrict__ actions, int ld,
                                                                   const float* __restrict__ v, int v_stride, int T,
                                                                   float* __restrict__ part, double* __restrict__ loss_part) {
    extern __shared__ float smem[];
    __shared__ double red[kTileWarps];
    float* const D0 = eupg_grad_buf(smem, sh, 0);
    const int L = sh.L, A = sh.w[L];
    const int c = blockIdx.x;
    int first, count;
    tile_range((T + kTileRows - 1) / kTileRows, c, first, count);
    const float inv_t = 1.0f / (float)T;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* out = part + (size_t)c * lay.total();
    double lsum = 0.0;  // lane 0 of each warp only

    for (int tile = first; tile < first + count; ++tile) {
        const bool init = tile == first;
        const int t0 = tile * kTileRows;
        eupg_stage(smem, sh, obs, acc, ld, t0, T);
        eupg_forward_tile(P, sh, smem, D0);

        // p, the clamped log-probability of the taken action, the loss term and dL/dz (one warp per row; A <= 32 so lane a holds z_a):
        //   dL/dz_a = g (1 - sigmoid(z_a)) ([a == action] - p_a),  g = -v / T where the clamp passes the gradient, else 0
        for (int r = warp; r < kTileRows; r += kTileWarps) {
            const int row = t0 + r;
            const bool valid = row < T;
            const float z = lane < A ? D0[r * A + lane] : 0.f;
            const float sg = lane < A ? sigmoid_f32(z) : 0.f;
            const float s = warp_sum_f32(sg);
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

        // backward, last layer first: dz_l is in gradient buffer `cur`; a_l (the input of layer l) is the tanh output of layer l - 1
        int cur = 0;
        for (int l = L - 1; l >= 0; --l) {
            tile_backward(P.p[2 * l], eupg_act(smem, sh, l), sh.w[l], eupg_grad_buf(smem, sh, cur), sh.w[l + 1], out + lay.offset(2 * l),
                          out + lay.offset(2 * l + 1), init, l > 0 ? eupg_grad_buf(smem, sh, cur ^ 1) : nullptr, Act::Tanh);
            cur ^= 1;
        }
    }

    // the other lanes hold +0.0, which leaves the lane-0 sums unchanged (lsum is never -0.0)
    const double lt = block_sum_f64<kTileThreads>(lsum, red);
    if (threadIdx.x == 0) loss_part[c] = lt;
}

// Block 0 of the partial sum: loss = -(sum of the CTAs' logp * v) / T.
struct EupgFinish {
    const double* loss_part;
    int T;
    float* loss_out;
    __device__ void operator()(int n_parts) const {
        if (threadIdx.x != 0) return;
        double l = 0.0;
        for (int c = 0; c < n_parts; ++c) l += loss_part[c];
        loss_out[0] = (float)(-l / (double)T);
    }
};

// Forward alone on N rows x [N, S + d]; out [N, A] = p.  x and out may live in mapped pinned host memory.
__global__ void __launch_bounds__(kTileThreads) eupg_probs_kernel(const __grid_constant__ EupgParams P,
                                                                  const __grid_constant__ EupgShape sh, const float* x, int N, float* out) {
    extern __shared__ float smem[];
    float* const D0 = eupg_grad_buf(smem, sh, 0);
    const int K = sh.w[0], A = sh.w[sh.L];
    const int r0 = blockIdx.x * kTileRows;
    const int nr = min(kTileRows, N - r0);
    for (int idx = threadIdx.x; idx < kTileRows * K; idx += kTileThreads) {
        const int r = idx / K;
        smem[idx] = r < nr ? x[(size_t)r0 * K + idx] : 0.f;
    }
    __syncthreads();
    eupg_forward_tile(P, sh, smem, D0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < nr; r += kTileWarps) {
        const float sg = lane < A ? sigmoid_f32(D0[r * A + lane]) : 0.f;
        const float s = warp_sum_f32(sg);
        if (lane < A) out[(size_t)(r0 + r) * A + lane] = sg / s;
    }
}

// c = gamma * c + r_t from t = T - 1 down to 0, per objective, with the product and the sum rounded separately.  CTA b owns objectives
// [256 b, 256 b + dc); its rewards are staged chunk by chunk (last chunk first) in shared memory, one thread per objective runs the
// recurrence, then the chunk is written out.  Objectives are independent, so any number of them is covered.
__global__ void __launch_bounds__(kEupgReturnsThreads) eupg_returns_kernel(const float* __restrict__ rewards, int ld, int T, int d, float gamma,
                                                                    float* __restrict__ out) {
    __shared__ float buf[kEupgReturnsSmem];
    const int k0 = blockIdx.x * kEupgReturnsThreads, dc = min(kEupgReturnsThreads, d - k0);
    const int chunk = kEupgReturnsSmem / dc;
    float c = 0.f;
    for (int hi = T; hi > 0; hi -= chunk) {
        const int lo = max(0, hi - chunk), n = hi - lo;
        for (int idx = threadIdx.x; idx < n * dc; idx += kEupgReturnsThreads) {
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
        for (int idx = threadIdx.x; idx < n * dc; idx += kEupgReturnsThreads) {
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

}  // namespace morl

extern "C" int morl_eupg_supported(int obs_dim, int d, const int* hidden, int n_hidden, int n_out) {
    morl::EupgShape sh;
    return morl::eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh) ? 1 : 0;
}

extern "C" size_t morl_eupg_workspace_bytes(int obs_dim, int d, const int* hidden, int n_hidden, int n_out) {
    using namespace morl;
    EupgShape sh;
    if (!eupg_shape(obs_dim, d, hidden, n_hidden, n_out, &sh)) return 0;
    return (size_t)kEupgCtas * sizeof(double) + (size_t)kEupgCtas * (size_t)sh.layout().total() * sizeof(float);
}

extern "C" int morl_eupg_returns_f32(const float* rewards, int ld, int T, int d, float gamma, float* out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(rewards && out, MORL_ERR_NULL, "morl_eupg_returns_f32: NULL pointer argument");
    MORL_REQUIRE(T > 0 && d > 0 && ld >= d, MORL_ERR_SHAPE, "morl_eupg_returns_f32: bad shape T=%d d=%d ld=%d", T, d, ld);
    eupg_returns_kernel<<<(d + kEupgReturnsThreads - 1) / kEupgReturnsThreads, kEupgReturnsThreads, 0, static_cast<cudaStream_t>(stream)>>>(rewards, ld, T, d, gamma, out);
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
    if (int rc = load_tables("morl_eupg_update_f32", 2 * sh.L, params, P, grads, &G)) return rc;
    const EupgLayout lay = sh.layout();
    const int ctas = min(kEupgCtas, (T + kTileRows - 1) / kTileRows);
    double* loss_part = static_cast<double*>(workspace);
    float* part = reinterpret_cast<float*>(loss_part + kEupgCtas);
    set_smem_limit_once<eupg_update_kernel>(eupg_max_smem_bytes());
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    eupg_update_kernel<<<ctas, kTileThreads, eupg_smem_floats(sh) * sizeof(float), st>>>(P, sh, lay, obs, acc, actions, ld, v, v_stride, T, part,
                                                                                        loss_part);
    launch_partial_sum(G, lay, part, ctas, EupgFinish{loss_part, T, loss_out}, st);
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
    if (int rc = load_tables("morl_eupg_probs_f32", 2 * sh.L, params, P)) return rc;
    set_smem_limit_once<eupg_probs_kernel>(eupg_max_smem_bytes());
    eupg_probs_kernel<<<(N + kTileRows - 1) / kTileRows, kTileThreads, eupg_smem_floats(sh) * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
        P, sh, x, N, out);
    return check_launch("morl_eupg_probs_f32");
}
