// pcn.cu -- the default PCN / LCN model (reference multi_policy/pcn/pcn.py:51-103) on CUDA cores.
//
//   c = [desired_return || horizon] * scaling,  s = sigmoid(Ls obs + bs),  e = sigmoid(Lc c + bc),
//   h = relu(W1 (s * e) + b1),  y = W2 h + b2,  log_softmax(y) for discrete actions, y as is for continuous ones.
//
// morl_pcn_update_f32  : minibatch gather from the episode store, forward, loss, backward (pcn.py:202-236) -- per-CTA gradient partials
//                        of a tile of kPcnRows rows, then a fixed-order sum over the tiles into the parameters' .grad storages
// morl_pcn_forward_f32 : the forward alone on N rows with their own commands (pcn.py:309-322 for one row), optional argmax
//
// The networks are tiny (hidden <= 256): one update is a few MFLOP and launch-bound, so the kernels favour few launches and fixed
// reduction orders over tensor cores.  Weights are read through the read-only cache; every activation of a tile lives in shared memory.
#include "common.cuh"

namespace morl {

constexpr int kPcnThreads = 256;
constexpr int kPcnRows = 16;  // rows per CTA
constexpr int kPcnMaxObs = 256;
constexpr int kPcnMaxA = 32;

// The rows a thread owns are g, g + groups, ... (rpt of them); the loop is unrolled to kPcnRows so that the per-row accumulators stay in
// registers.
#define MORL_PCN_ROWS(i) _Pragma("unroll") for (int i = 0; i < kPcnRows; ++i) if (i < rpt)

struct PcnParams {
    const float* p[8];  // Ls [H, S], bs [H], Lc [H, d + 1], bc [H], W1 [H, H], b1 [H], W2 [A, H], b2 [A]
};
struct PcnGrads {
    float* g[8];
};

struct PcnShape {
    int S, D1, H, A;
    __host__ __device__ int size(int t) const {
        switch (t) {
            case 0: return H * S;
            case 1: return H;
            case 2: return H * D1;
            case 3: return H;
            case 4: return H * H;
            case 5: return H;
            case 6: return A * H;
            default: return A;
        }
    }
    __host__ __device__ int offset(int t) const {
        int o = 0;
        for (int i = 0; i < t; ++i) o += size(i);
        return o;
    }
    __host__ __device__ int total() const { return offset(8); }
};

struct PcnSmem {
    float *obs, *c, *s, *e, *x, *h, *dh, *y;
};

__host__ __device__ inline size_t pcn_smem_floats(const PcnShape& sh) {
    return (size_t)kPcnRows * (sh.S + sh.D1 + 5 * sh.H + sh.A);
}

__device__ inline PcnSmem pcn_carve(float* base, const PcnShape& sh) {
    PcnSmem m;
    m.obs = base;
    m.c = m.obs + kPcnRows * sh.S;
    m.s = m.c + kPcnRows * sh.D1;
    m.e = m.s + kPcnRows * sh.H;
    m.x = m.e + kPcnRows * sh.H;
    m.h = m.x + kPcnRows * sh.H;
    m.dh = m.h + kPcnRows * sh.H;
    m.y = m.dh + kPcnRows * sh.H;
    return m;
}

__device__ __forceinline__ float sigmoidf_(float z) { return 1.0f / (1.0f + expf(-z)); }

// s, e, x = s * e, h, y of the tile's rows (obs and c already staged).  Thread j of each row group walks weight row j once and
// applies it to its rows (kPcnRows * H / kPcnThreads of them), so every weight load is reused across the rows from registers.
__device__ void pcn_forward_tile(const PcnParams& P, const PcnShape& sh, const PcnSmem& m) {
    const int H = sh.H, S = sh.S, D1 = sh.D1, A = sh.A;
    const int groups = kPcnThreads / H, j = threadIdx.x % H, g = threadIdx.x / H;
    const int rpt = kPcnRows / groups;
    {
        float as[kPcnRows], ae[kPcnRows];
        const float bs = __ldg(P.p[1] + j), bc = __ldg(P.p[3] + j);
        MORL_PCN_ROWS(i) as[i] = 0.f, ae[i] = 0.f;
        const float* ls = P.p[0] + (size_t)j * S;
        for (int k = 0; k < S; ++k) {
            const float w = __ldg(ls + k);
            MORL_PCN_ROWS(i) as[i] = fmaf(w, m.obs[(g + groups * i) * S + k], as[i]);
        }
        const float* lc = P.p[2] + (size_t)j * D1;
        for (int k = 0; k < D1; ++k) {
            const float w = __ldg(lc + k);
            MORL_PCN_ROWS(i) ae[i] = fmaf(w, m.c[(g + groups * i) * D1 + k], ae[i]);
        }
        MORL_PCN_ROWS(i) {
            const int r = g + groups * i;
            const float s = sigmoidf_(as[i] + bs), e = sigmoidf_(ae[i] + bc);
            m.s[r * H + j] = s;
            m.e[r * H + j] = e;
            m.x[r * H + j] = s * e;
        }
    }
    __syncthreads();
    {
        float ah[kPcnRows];
        const float b1 = __ldg(P.p[5] + j);
        MORL_PCN_ROWS(i) ah[i] = 0.f;
        const float* w1 = P.p[4] + (size_t)j * H;
        for (int k = 0; k < H; ++k) {
            const float w = __ldg(w1 + k);
            MORL_PCN_ROWS(i) ah[i] = fmaf(w, m.x[(g + groups * i) * H + k], ah[i]);
        }
        MORL_PCN_ROWS(i) m.h[(g + groups * i) * H + j] = fmaxf(ah[i] + b1, 0.f);
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < kPcnRows * A; idx += kPcnThreads) {
        const int r = idx / A, a = idx % A;
        const float* w2 = P.p[6] + (size_t)a * H;
        const float* hr = m.h + r * H;
        float acc = 0.f;
        for (int k = 0; k < H; ++k) acc = fmaf(__ldg(w2 + k), hr[k], acc);
        m.y[r * A + a] = acc + __ldg(P.p[7] + a);
    }
    __syncthreads();
}

// log_softmax of the tile's rows in place (one warp per row; A <= 32 so lane a holds y[a]): (y - max) - log(sum exp(y - max))
__device__ void pcn_log_softmax_tile(const PcnShape& sh, const PcnSmem& m) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, A = sh.A;
    for (int r = warp; r < kPcnRows; r += kPcnThreads / 32) {
        const float v = lane < A ? m.y[r * A + lane] : -INFINITY;
        float mx = v;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float z = v - mx;
        float se = lane < A ? expf(z) : 0.f;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) se += __shfl_xor_sync(0xffffffffu, se, off);
        if (lane < A) m.y[r * A + lane] = z - logf(se);
    }
    __syncthreads();
}

__device__ __forceinline__ double pcn_block_sum(double v, double* red) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < kPcnThreads / 32; ++i) t += red[i];
    return t;
}

// One tile of kPcnRows minibatch rows: gather, forward, loss, backward; writes this CTA's gradient partials (every parameter element,
// summed over the tile's rows in row order) and its loss / entropy partials.
__global__ void __launch_bounds__(kPcnThreads) pcn_update_kernel(PcnParams P, PcnShape sh, const float* __restrict__ scaling,
                                                                 const float* __restrict__ store, int ld, const int32_t* __restrict__ rows,
                                                                 const int32_t* __restrict__ horizons, int B, int continuous,
                                                                 float* __restrict__ pred_out, float* __restrict__ part,
                                                                 double* __restrict__ loss_part) {
    extern __shared__ float smem[];
    __shared__ double red[kPcnThreads / 32];
    const PcnSmem m = pcn_carve(smem, sh);
    const int S = sh.S, D1 = sh.D1, H = sh.H, A = sh.A, d = D1 - 1;
    const int r0 = blockIdx.x * kPcnRows;
    const int nr = min(kPcnRows, B - r0);

    // prologue: gather obs and [return-to-go || horizon] * scaling of the tile's rows (rows past the batch are zero)
    for (int idx = threadIdx.x; idx < kPcnRows * S; idx += kPcnThreads) {
        const int r = idx / S, k = idx % S;
        m.obs[idx] = r < nr ? __ldg(store + (size_t)__ldg(rows + r0 + r) * ld + k) : 0.f;
    }
    for (int idx = threadIdx.x; idx < kPcnRows * D1; idx += kPcnThreads) {
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
    for (int idx = threadIdx.x; idx < kPcnRows * A; idx += kPcnThreads) {
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
    const double lsum = pcn_block_sum(l_part, red);
    const double esum = pcn_block_sum(e_part, red);
    if (threadIdx.x == 0) {
        loss_part[2 * blockIdx.x] = lsum;
        loss_part[2 * blockIdx.x + 1] = esum;
    }
    __syncthreads();

    float* out = part + (size_t)blockIdx.x * sh.total();
    // W2, b2
    {
        float* gw = out + sh.offset(6);
        for (int idx = threadIdx.x; idx < A * H; idx += kPcnThreads) {
            const int a = idx / H, k = idx % H;
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc = fmaf(m.y[r * A + a], m.h[r * H + k], acc);
            gw[idx] = acc;
        }
        float* gb = out + sh.offset(7);
        for (int a = threadIdx.x; a < A; a += kPcnThreads) {
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc += m.y[r * A + a];
            gb[a] = acc;
        }
    }
    // dh = (h > 0) * W2^T dy
    const int groups = kPcnThreads / H, j = threadIdx.x % H, g = threadIdx.x / H;
    const int rpt = kPcnRows / groups;
    MORL_PCN_ROWS(i) {
        const int r = g + groups * i;
        float acc = 0.f;
        for (int a = 0; a < A; ++a) acc = fmaf(__ldg(P.p[6] + (size_t)a * H + j), m.y[r * A + a], acc);
        m.dh[r * H + j] = m.h[r * H + j] > 0.f ? acc : 0.f;
    }
    __syncthreads();
    // W1, b1
    {
        float* gw = out + sh.offset(4);
        for (int idx = threadIdx.x; idx < H * H; idx += kPcnThreads) {
            const int jj = idx / H, k = idx % H;
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc = fmaf(m.dh[r * H + jj], m.x[r * H + k], acc);
            gw[idx] = acc;
        }
        float* gb = out + sh.offset(5);
        for (int jj = threadIdx.x; jj < H; jj += kPcnThreads) {
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc += m.dh[r * H + jj];
            gb[jj] = acc;
        }
    }
    // dx = W1^T dh, then through x = s * e and the two sigmoids: s and e become the pre-activation gradients dzs and dze
    {
        float ax[kPcnRows];
        MORL_PCN_ROWS(i) ax[i] = 0.f;
        for (int jj = 0; jj < H; ++jj) {
            const float w = __ldg(P.p[4] + (size_t)jj * H + j);
            MORL_PCN_ROWS(i) ax[i] = fmaf(w, m.dh[(g + groups * i) * H + jj], ax[i]);
        }
        MORL_PCN_ROWS(i) {
            const int r = g + groups * i;
            const float s = m.s[r * H + j], e = m.e[r * H + j];
            m.s[r * H + j] = ax[i] * e * (1.f - s) * s;
            m.e[r * H + j] = ax[i] * s * (1.f - e) * e;
        }
    }
    __syncthreads();
    // Ls, bs, Lc, bc
    {
        float* gls = out + sh.offset(0);
        for (int idx = threadIdx.x; idx < H * S; idx += kPcnThreads) {
            const int jj = idx / S, k = idx % S;
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc = fmaf(m.s[r * H + jj], m.obs[r * S + k], acc);
            gls[idx] = acc;
        }
        float* glc = out + sh.offset(2);
        for (int idx = threadIdx.x; idx < H * D1; idx += kPcnThreads) {
            const int jj = idx / D1, k = idx % D1;
            float acc = 0.f;
            for (int r = 0; r < kPcnRows; ++r) acc = fmaf(m.e[r * H + jj], m.c[r * D1 + k], acc);
            glc[idx] = acc;
        }
        float* gbs = out + sh.offset(1);
        float* gbc = out + sh.offset(3);
        for (int jj = threadIdx.x; jj < H; jj += kPcnThreads) {
            float as = 0.f, ae = 0.f;
            for (int r = 0; r < kPcnRows; ++r) as += m.s[r * H + jj], ae += m.e[r * H + jj];
            gbs[jj] = as;
            gbc[jj] = ae;
        }
    }
}

// Fixed-order sum of the tiles' partials into the eight .grad storages; block 0 also finishes the loss and the entropy.
__global__ void __launch_bounds__(kPcnThreads) pcn_reduce_kernel(PcnGrads G, PcnShape sh, const float* __restrict__ part,
                                                                 const double* __restrict__ loss_part, int n_tiles, int B, int continuous,
                                                                 float* __restrict__ loss_out, float* __restrict__ entropy_out) {
    const int total = sh.total();
    int off = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {  // unrolled: G.g[k] stays a kernel parameter, not a stack array
        const int n = sh.size(k);
        for (int q = blockIdx.x * kPcnThreads + threadIdx.x; q < n; q += gridDim.x * kPcnThreads) {
            float acc = 0.f;
            for (int t = 0; t < n_tiles; ++t) acc += __ldg(part + (size_t)t * total + off + q);
            G.g[k][q] = acc;
        }
        off += n;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        double l = 0.0, e = 0.0;
        for (int t = 0; t < n_tiles; ++t) l += loss_part[2 * t], e += loss_part[2 * t + 1];
        loss_out[0] = (float)(continuous ? l / ((double)B * sh.A) : l / (double)B);
        if (entropy_out) entropy_out[0] = (float)e;
    }
}

// Forward alone on N rows (obs [N, S], ret [N, d], hor [N]; any of them, and out / argmax_out, may live in mapped pinned host memory).
__global__ void __launch_bounds__(kPcnThreads) pcn_forward_kernel(PcnParams P, PcnShape sh, const float* __restrict__ scaling,
                                                                  const float* obs, const float* ret, const float* hor, int N, int log_softmax,
                                                                  float* out, int32_t* argmax_out) {
    extern __shared__ float smem[];
    const PcnSmem m = pcn_carve(smem, sh);
    const int S = sh.S, D1 = sh.D1, A = sh.A, d = D1 - 1;
    const int r0 = blockIdx.x * kPcnRows;
    const int nr = min(kPcnRows, N - r0);
    for (int idx = threadIdx.x; idx < kPcnRows * S; idx += kPcnThreads) {
        const int r = idx / S, k = idx % S;
        m.obs[idx] = r < nr ? obs[(size_t)(r0 + r) * S + k] : 0.f;
    }
    for (int idx = threadIdx.x; idx < kPcnRows * D1; idx += kPcnThreads) {
        const int r = idx / D1, k = idx % D1;
        float v = 0.f;
        if (r < nr) v = k < d ? ret[(size_t)(r0 + r) * d + k] : hor[r0 + r];
        m.c[idx] = v * __ldg(scaling + k);
    }
    __syncthreads();
    pcn_forward_tile(P, sh, m);
    if (log_softmax) pcn_log_softmax_tile(sh, m);
    for (int idx = threadIdx.x; idx < nr * A; idx += kPcnThreads) out[(size_t)(r0 + idx / A) * A + idx % A] = m.y[idx];
    if (argmax_out) {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int r = warp; r < nr; r += kPcnThreads / 32) {
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

static int pcn_tiles(int B) { return (B + kPcnRows - 1) / kPcnRows; }

}  // namespace morl

extern "C" int morl_pcn_supported(int obs_dim, int d, int hidden, int n_out, int batch) {
    return morl::pcn_shape_ok(obs_dim, d, hidden, n_out) && batch >= 1 && batch <= MORL_PCN_MAX_BATCH ? 1 : 0;
}

extern "C" size_t morl_pcn_workspace_bytes(int obs_dim, int d, int hidden, int n_out, int batch) {
    using namespace morl;
    if (!morl_pcn_supported(obs_dim, d, hidden, n_out, batch)) return 0;
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const size_t tiles = (size_t)pcn_tiles(batch);
    return tiles * 2 * sizeof(double) + tiles * (size_t)sh.total() * sizeof(float);
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
    for (int t = 0; t < 8; ++t) {
        MORL_REQUIRE(params[t] && grads[t], MORL_ERR_NULL, "morl_pcn_update_f32: NULL parameter or gradient pointer %d", t);
        P.p[t] = params[t];
        G.g[t] = grads[t];
    }
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const int tiles = pcn_tiles(B);
    double* loss_part = static_cast<double*>(workspace);
    float* part = reinterpret_cast<float*>(loss_part + 2 * (size_t)tiles);
    const size_t smem = pcn_smem_floats(sh) * sizeof(float);
    set_smem_limit_once<pcn_update_kernel>(pcn_smem_floats(PcnShape{kPcnMaxObs, MORL_MAX_D + 1, 256, kPcnMaxA}) * sizeof(float));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    pcn_update_kernel<<<tiles, kPcnThreads, smem, st>>>(P, sh, scaling, store, ld_store, rows, horizons, B, continuous ? 1 : 0,
                                                         pred_out, part, loss_part);
    const int rblocks = min((sh.total() + kPcnThreads - 1) / kPcnThreads, 4 * sm_count());
    pcn_reduce_kernel<<<rblocks, kPcnThreads, 0, st>>>(G, sh, part, loss_part, tiles, B, continuous ? 1 : 0, loss_out,
                                                        continuous ? nullptr : entropy_out);
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
    for (int t = 0; t < 8; ++t) {
        MORL_REQUIRE(params[t], MORL_ERR_NULL, "morl_pcn_forward_f32: NULL parameter pointer %d", t);
        P.p[t] = params[t];
    }
    const PcnShape sh{obs_dim, d + 1, hidden, n_out};
    const size_t smem = pcn_smem_floats(sh) * sizeof(float);
    set_smem_limit_once<pcn_forward_kernel>(pcn_smem_floats(PcnShape{kPcnMaxObs, MORL_MAX_D + 1, 256, kPcnMaxA}) * sizeof(float));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    pcn_forward_kernel<<<pcn_tiles(N), kPcnThreads, smem, st>>>(P, sh, scaling, obs, ret, hor, N, log_softmax ? 1 : 0, out, argmax_out);
    return check_launch("morl_pcn_forward_f32");
}
