// pcn.cu -- the default PCN / LCN model (reference multi_policy/pcn/pcn.py:51-103) on CUDA cores.
//
//   c = [desired_return || horizon] * scaling,  s = sigmoid(Ls obs + bs),  e = sigmoid(Lc c + bc),
//   h = relu(W1 (s * e) + b1),  y = W2 h + b2,  log_softmax(y) for discrete actions, y as is for continuous ones.
//
// morl_pcn_update_f32  : minibatch gather from the episode store, forward, loss, backward (pcn.py:202-236) -- per-CTA gradient partials
//                        of a tile of 16 rows, then a fixed-order sum over the tiles into the parameters' .grad storages
// morl_pcn_forward_f32 : the forward alone on N rows with their own commands (pcn.py:309-322 for one row), optional argmax
//
// The networks are tiny (hidden <= 256): one update is a few MFLOP and launch-bound, so the kernels favour few launches and fixed
// reduction orders over tensor cores.  Weights are read through the read-only cache; every activation of a tile lives in shared memory.
#include "tile_mlp.cuh"

namespace morl {

constexpr int kPcnMaxObs = 256;
constexpr int kPcnMaxA = 32;

using PcnParams = ParamTable<8>;  // Ls [H, S], bs [H], Lc [H, d + 1], bc [H], W1 [H, H], b1 [H], W2 [A, H], b2 [A]
using PcnGrads = GradTable<8>;
using PcnLayout = ParamLayout<8>;

struct PcnShape {
    int S, D1, H, A;
    PcnLayout layout() const { return PcnLayout{8, {H * S, H, H * D1, H, H * H, H, A * H, A}}; }
};

struct PcnSmem {
    float *obs, *c, *s, *e, *x, *h, *dh, *y;
};

__host__ __device__ inline size_t pcn_smem_floats(const PcnShape& sh) {
    return (size_t)kTileRows * (sh.S + sh.D1 + 5 * sh.H + sh.A);
}

__device__ inline PcnSmem pcn_carve(float* base, const PcnShape& sh) {
    PcnSmem m;
    m.obs = base;
    m.c = m.obs + kTileRows * sh.S;
    m.s = m.c + kTileRows * sh.D1;
    m.e = m.s + kTileRows * sh.H;
    m.x = m.e + kTileRows * sh.H;
    m.h = m.x + kTileRows * sh.H;
    m.dh = m.h + kTileRows * sh.H;
    m.y = m.dh + kTileRows * sh.H;
    return m;
}

// s, e, x = s * e, h, y of the tile's rows (obs and c already staged).
__device__ void pcn_forward_tile(const PcnParams& P, const PcnShape& sh, const PcnSmem& m) {
    const int H = sh.H;
    tile_linear(P.p[0], P.p[1], m.obs, sh.S, m.s, H, Act::Sigmoid);
    tile_linear(P.p[2], P.p[3], m.c, sh.D1, m.e, H, Act::Sigmoid);
    for (int idx = threadIdx.x; idx < kTileRows * H; idx += kTileThreads) m.x[idx] = m.s[idx] * m.e[idx];
    __syncthreads();
    tile_linear(P.p[4], P.p[5], m.x, H, m.h, H, Act::Relu);
    tile_linear(P.p[6], P.p[7], m.h, H, m.y, sh.A, Act::None);
}

// log_softmax of the tile's rows in place (one warp per row; A <= 32 so lane a holds y[a]): (y - max) - log(sum exp(y - max))
__device__ void pcn_log_softmax_tile(const PcnShape& sh, const PcnSmem& m) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, A = sh.A;
    for (int r = warp; r < kTileRows; r += kTileWarps) {
        const float v = lane < A ? m.y[r * A + lane] : -INFINITY;
        const float z = v - warp_max_f32(v);
        const float se = warp_sum_f32(lane < A ? expf(z) : 0.f);
        if (lane < A) m.y[r * A + lane] = z - logf(se);
    }
    __syncthreads();
}

// One tile of kTileRows minibatch rows: gather, forward, loss, backward; writes this CTA's gradient partials (every parameter element,
// summed over the tile's rows in row order) and its loss / entropy partials.
__global__ void __launch_bounds__(kTileThreads) pcn_update_kernel(PcnParams P, PcnShape sh, const __grid_constant__ PcnLayout lay,
                                                                  const float* __restrict__ scaling,
                                                                 const float* __restrict__ store, int ld, const int32_t* __restrict__ rows,
                                                                 const int32_t* __restrict__ horizons, int B, int continuous,
                                                                 float* __restrict__ pred_out, float* __restrict__ part,
                                                                 double* __restrict__ loss_part) {
    extern __shared__ float smem[];
    __shared__ double red[kTileWarps];
    const PcnSmem m = pcn_carve(smem, sh);
    const int S = sh.S, D1 = sh.D1, H = sh.H, A = sh.A, d = D1 - 1;
    const int r0 = blockIdx.x * kTileRows;
    const int nr = min(kTileRows, B - r0);

    // prologue: gather obs and [return-to-go || horizon] * scaling of the tile's rows (rows past the batch are zero)
    for (int idx = threadIdx.x; idx < kTileRows * S; idx += kTileThreads) {
        const int r = idx / S, k = idx % S;
        m.obs[idx] = r < nr ? __ldg(store + (size_t)__ldg(rows + r0 + r) * ld + k) : 0.f;
    }
    for (int idx = threadIdx.x; idx < kTileRows * D1; idx += kTileThreads) {
        const int r = idx / D1, k = idx % D1;
        float v = 0.f;
        if (r < nr) v = k < d ? __ldg(store + (size_t)__ldg(rows + r0 + r) * ld + S + k) : (float)__ldg(horizons + r0 + r);
        m.c[idx] = v * __ldg(scaling + k);
    }
    __syncthreads();
    pcn_forward_tile(P, sh, m);
    if (!continuous) pcn_log_softmax_tile(sh, m);

    // loss, entropy and dL/dy (m.y becomes dy once the prediction is written out)
    double l_part = 0.0, e_part = 0.0;
    const float inv_b = 1.0f / (float)B;
    const float inv_ba = 2.0f / ((float)B * (float)A);
    for (int idx = threadIdx.x; idx < kTileRows * A; idx += kTileThreads) {
        const int r = idx / A, a = idx % A;
        float dy = 0.f;
        if (r < nr) {
            const float y = m.y[idx];
            const float* act = store + (size_t)__ldg(rows + r0 + r) * ld + S + d;
            if (pred_out) pred_out[(size_t)(r0 + r) * A + a] = y;
            if (continuous) {
                const float diff = y - __ldg(act + a);
                l_part += (double)(diff * diff);
                dy = diff * inv_ba;
            } else {
                const float p = expf(y);
                const bool hit = __ldg(reinterpret_cast<const int32_t*>(act)) == a;
                if (hit) l_part -= (double)y;
                e_part -= (double)(p * y);
                dy = (p - (hit ? 1.f : 0.f)) * inv_b;
            }
        }
        m.y[idx] = dy;
    }
    const double lsum = block_sum_f64<kTileThreads>(l_part, red);
    const double esum = block_sum_f64<kTileThreads>(e_part, red);
    if (threadIdx.x == 0) {
        loss_part[2 * blockIdx.x] = lsum;
        loss_part[2 * blockIdx.x + 1] = esum;
    }
    __syncthreads();

    float* out = part + (size_t)blockIdx.x * lay.total();
    // W2, b2 and dh = (h > 0) W2^T dy
    tile_backward(P.p[6], m.h, H, m.y, A, out + lay.offset(6), out + lay.offset(7), true, m.dh, Act::Relu);
    // W1, b1 and dx = W1^T dh into m.h (h is dead once the ReLU mask has been applied)
    tile_backward(P.p[4], m.x, H, m.dh, H, out + lay.offset(4), out + lay.offset(5), true, m.h, Act::None);
    // through x = s * e and the two sigmoids: s and e become the pre-activation gradients dzs and dze
    for (int idx = threadIdx.x; idx < kTileRows * H; idx += kTileThreads) {
        const float dx = m.h[idx], s = m.s[idx], e = m.e[idx];
        m.s[idx] = dx * e * (1.f - s) * s;
        m.e[idx] = dx * s * (1.f - e) * e;
    }
    __syncthreads();
    // Ls, bs, Lc, bc
    tile_backward(P.p[0], m.obs, S, m.s, H, out + lay.offset(0), out + lay.offset(1), true, nullptr, Act::None);
    tile_backward(P.p[2], m.c, D1, m.e, H, out + lay.offset(2), out + lay.offset(3), true, nullptr, Act::None);
}

// Block 0 of the partial sum: the loss and the batch entropy from the tiles' partials.
struct PcnFinish {
    const double* loss_part;
    int B, A, continuous;
    float* loss_out;
    float* entropy_out;
    __device__ void operator()(int n_tiles) const {
        if (threadIdx.x != 0) return;
        double l = 0.0, e = 0.0;
        for (int t = 0; t < n_tiles; ++t) l += loss_part[2 * t], e += loss_part[2 * t + 1];
        loss_out[0] = (float)(continuous ? l / ((double)B * A) : l / (double)B);
        if (entropy_out) entropy_out[0] = (float)e;
    }
};

// Forward alone on N rows (obs [N, S], ret [N, d], hor [N]; any of them, and out / argmax_out, may live in mapped pinned host memory).
__global__ void __launch_bounds__(kTileThreads) pcn_forward_kernel(PcnParams P, PcnShape sh, const float* __restrict__ scaling,
                                                                  const float* obs, const float* ret, const float* hor, int N, int log_softmax,
                                                                  float* out, int32_t* argmax_out) {
    extern __shared__ float smem[];
    const PcnSmem m = pcn_carve(smem, sh);
    const int S = sh.S, D1 = sh.D1, A = sh.A, d = D1 - 1;
    const int r0 = blockIdx.x * kTileRows;
    const int nr = min(kTileRows, N - r0);
    for (int idx = threadIdx.x; idx < kTileRows * S; idx += kTileThreads) {
        const int r = idx / S, k = idx % S;
        m.obs[idx] = r < nr ? obs[(size_t)(r0 + r) * S + k] : 0.f;
    }
    for (int idx = threadIdx.x; idx < kTileRows * D1; idx += kTileThreads) {
        const int r = idx / D1, k = idx % D1;
        float v = 0.f;
        if (r < nr) v = k < d ? ret[(size_t)(r0 + r) * d + k] : hor[r0 + r];
        m.c[idx] = v * __ldg(scaling + k);
    }
    __syncthreads();
    pcn_forward_tile(P, sh, m);
    if (log_softmax) pcn_log_softmax_tile(sh, m);
    for (int idx = threadIdx.x; idx < nr * A; idx += kTileThreads) out[(size_t)(r0 + idx / A) * A + idx % A] = m.y[idx];
    if (argmax_out) {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int r = warp; r < nr; r += kTileWarps) {
            float v = lane < A ? m.y[r * A + lane] : -INFINITY;
            int i = lane < A ? lane : 0x7fffffff;
            warp_argmax(v, i);
            if (lane == 0) argmax_out[r0 + r] = i;
        }
    }
}

static bool pcn_shape_ok(int S, int d, int H, int A) {
    return S >= 1 && S <= kPcnMaxObs && d >= 1 && d <= MORL_MAX_D && (H == 32 || H == 64 || H == 128 || H == 256) && A >= 1 && A <= kPcnMaxA;
}

static int pcn_tiles(int B) { return (B + kTileRows - 1) / kTileRows; }

}  // namespace morl

extern "C" int morl_pcn_supported(int obs_dim, int d, int hidden, int n_out, int batch) {
    return morl::pcn_shape_ok(obs_dim, d, hidden, n_out) && batch >= 1 && batch <= MORL_PCN_MAX_BATCH ? 1 : 0;
}

extern "C" size_t morl_pcn_workspace_bytes(int obs_dim, int d, int hidden, int n_out, int batch) {
    using namespace morl;
    if (!morl_pcn_supported(obs_dim, d, hidden, n_out, batch)) return 0;
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const size_t tiles = (size_t)pcn_tiles(batch);
    return tiles * 2 * sizeof(double) + tiles * (size_t)sh.layout().total() * sizeof(float);
}

extern "C" int morl_pcn_update_f32(const float* const* params, float* const* grads, const float* scaling, const float* store, int ld_store,
                                   const int32_t* rows, const int32_t* horizons, int B,
                                   int obs_dim, int d, int hidden, int n_out, int continuous, float* loss_out, float* entropy_out,
                                   float* pred_out, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && grads && scaling && store && rows && horizons && loss_out && workspace, MORL_ERR_NULL,
                 "morl_pcn_update_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && obs_dim > 0 && d > 0 && hidden > 0 && n_out > 0, MORL_ERR_SHAPE, "morl_pcn_update_f32: bad shape B=%d S=%d d=%d H=%d A=%d",
                 B, obs_dim, d, hidden, n_out);
    MORL_REQUIRE(morl_pcn_supported(obs_dim, d, hidden, n_out, B), MORL_ERR_UNSUPPORTED,
                 "morl_pcn_update_f32: unsupported configuration S=%d d=%d H=%d A=%d B=%d (morl_pcn_supported)", obs_dim, d, hidden, n_out, B);
    MORL_REQUIRE(ld_store >= obs_dim + d + (continuous ? n_out : 1), MORL_ERR_SHAPE, "morl_pcn_update_f32: ld_store=%d < S + d + action columns",
                 ld_store);
    PcnParams P;
    PcnGrads G;
    if (int rc = load_tables("morl_pcn_update_f32", 8, params, P, grads, &G)) return rc;
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const PcnLayout lay = sh.layout();
    const int tiles = pcn_tiles(B);
    double* loss_part = static_cast<double*>(workspace);
    float* part = reinterpret_cast<float*>(loss_part + 2 * (size_t)tiles);
    const size_t smem = pcn_smem_floats(sh) * sizeof(float);
    set_smem_limit_once<pcn_update_kernel>(pcn_smem_floats(PcnShape{kPcnMaxObs, MORL_MAX_D + 1, 256, kPcnMaxA}) * sizeof(float));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    pcn_update_kernel<<<tiles, kTileThreads, smem, st>>>(P, sh, lay, scaling, store, ld_store, rows, horizons, B, continuous ? 1 : 0,
                                                         pred_out, part, loss_part);
    launch_partial_sum(G, lay, part, tiles, PcnFinish{loss_part, B, n_out, continuous ? 1 : 0, loss_out, continuous ? nullptr : entropy_out}, st);
    return check_launch("morl_pcn_update_f32");
}

extern "C" int morl_pcn_forward_f32(const float* const* params, const float* scaling, const float* obs, const float* ret, const float* hor, int N,
                                    int obs_dim, int d, int hidden, int n_out, int log_softmax, float* out, int32_t* argmax_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && scaling && obs && ret && hor && out, MORL_ERR_NULL, "morl_pcn_forward_f32: NULL pointer argument");
    MORL_REQUIRE(N > 0 && obs_dim > 0 && d > 0 && hidden > 0 && n_out > 0, MORL_ERR_SHAPE, "morl_pcn_forward_f32: bad shape N=%d S=%d d=%d H=%d A=%d",
                 N, obs_dim, d, hidden, n_out);
    MORL_REQUIRE(pcn_shape_ok(obs_dim, d, hidden, n_out), MORL_ERR_UNSUPPORTED,
                 "morl_pcn_forward_f32: unsupported configuration S=%d d=%d H=%d A=%d (morl_pcn_supported)", obs_dim, d, hidden, n_out);
    PcnParams P;
    if (int rc = load_tables("morl_pcn_forward_f32", 8, params, P)) return rc;
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const size_t smem = pcn_smem_floats(sh) * sizeof(float);
    set_smem_limit_once<pcn_forward_kernel>(pcn_smem_floats(PcnShape{kPcnMaxObs, MORL_MAX_D + 1, 256, kPcnMaxA}) * sizeof(float));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    pcn_forward_kernel<<<pcn_tiles(N), kTileThreads, smem, st>>>(P, sh, scaling, obs, ret, hor, N, log_softmax ? 1 : 0, out, argmax_out);
    return check_launch("morl_pcn_forward_f32");
}
