// optim.cu -- multi-tensor target-network sync (SURVEY.md K11).
//
// Replaces polyak_update (reference common/networks.py:121-139), which issues 1-2 tiny kernels per parameter tensor
// (10 tensors for the Envelope Q-net, 2 nets x ~14 tensors for GPI-PD), with ONE launch over a device-side table of
// (param, target, size) entries.  Arithmetic is the reference's: tau == 1 -> copy, else
//   target.mul_(1 - tau); th.add(target, param, alpha=tau, out=target)    i.e.   fma(tau, p, fl(t * (1 - tau)))
// (ATen's CPU add-with-alpha kernel is a vectorised fmadd -- probed bit-exact in the build container, DESIGN.md).
#include "common.cuh"

namespace morl {

__global__ void __launch_bounds__(256) polyak_kernel(const float* const* __restrict__ params, float* const* __restrict__ targets,
                                                     const int64_t* __restrict__ sizes, float tau, float one_minus_tau) {
    pdl_enter();
    const int t = blockIdx.y;
    const int64_t n = sizes[t];
    const float* __restrict__ p = params[t];
    float* __restrict__ q = targets[t];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        if (tau == 1.0f)
            q[e] = p[e];
        else
            q[e] = __fmaf_rn(tau, p[e], __fmul_rn(q[e], one_minus_tau));
    }
}

}  // namespace morl

extern "C" int morl_polyak_f32(const float* const* params, float* const* targets, const int64_t* sizes, int n_tensors, int64_t max_size,
                               double tau, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && targets && sizes, MORL_ERR_NULL, "morl_polyak_f32: NULL pointer argument");
    MORL_REQUIRE(n_tensors > 0 && n_tensors <= 65535 && max_size > 0, MORL_ERR_SHAPE, "morl_polyak_f32: bad n_tensors=%d max_size=%lld",
                 n_tensors, (long long)max_size);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    long long bx = (max_size + 255) / 256;
    if (bx > 132 * 4) bx = 132 * 4;
    const dim3 grid((unsigned)bx, (unsigned)n_tensors, 1);
    // (1 - tau) is formed in double then rounded, like Python's `1.0 - tau` handed to Tensor.mul_
    const float omt = (float)(1.0 - tau);
    launch_k(polyak_kernel, dim3(grid), dim3(256), 0, st, params, targets, sizes, (float)tau, omt);
    return check_launch("morl_polyak_f32");
}

// ---- fused gradient clipping + Adam (SURVEY.md K11 / 8(f) item 2) ----------------------------------------------------------
// Replaces th.nn.utils.clip_grad_norm_ + optim.Adam.step (reference multi_policy/envelope/envelope.py:324-326): ~25 foreach /
// elementwise launches over 10 small tensors become two launches.  Arithmetic is the reference's non-capturable
// single-tensor Adam (torch/optim/adam.py, _single_tensor_adam): m <- lerp(m, g, 1-b1); v <- v*b2 + (1-b2) g^2;
// p <- p - (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps), with 1 - b^t evaluated in double like Python does;
// the clip coefficient is min(1, max_norm / (||g||_2 + 1e-6)) over ALL tensors (clip_grad_norm_ semantics).
namespace morl {

constexpr int kOptBlock = 256;

__global__ void __launch_bounds__(kOptBlock) grad_sqnorm_kernel(const float* const* __restrict__ grads, const int64_t* __restrict__ sizes,
                                                                float* const* __restrict__ steps, float* __restrict__ partials) {
    pdl_enter();
    __shared__ float red[kOptBlock / 32];
    const int t = blockIdx.y;
    const int64_t n = sizes[t];
    const float* __restrict__ g = grads[t];
    float acc = 0.f;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) acc += g[e] * g[e];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kOptBlock / 32; ++w) s += red[w];
        partials[(size_t)t * gridDim.x + blockIdx.x] = s;
        if (blockIdx.x == 0) *steps[t] += 1.0f;  // optimiser step counter of this tensor (read by adam_clip_kernel, same stream)
    }
}

__global__ void __launch_bounds__(kOptBlock) adam_clip_kernel(float* const* __restrict__ params, const float* const* __restrict__ grads,
                                                              float* const* __restrict__ exp_avg, float* const* __restrict__ exp_avg_sq,
                                                              float* const* __restrict__ steps, const int64_t* __restrict__ sizes,
                                                              const float* __restrict__ partials, int n_partials, float max_norm, float lr,
                                                              const double* __restrict__ lr_dev, float beta1, float beta2, float eps) {
    pdl_enter();
    __shared__ float s_coef;
    __shared__ double s_red[kOptBlock / 32];
    if (max_norm > 0.f) {
        // total squared norm: every block re-reduces the (few hundred) partials with the whole block, in a fixed tree order
        // (deterministic); a single thread walking them serially was ~10 us of latency in front of every block
        double tot = 0.0;
        for (int i = threadIdx.x; i < n_partials; i += kOptBlock) tot += (double)partials[i];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = tot;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t2 = 0.0;
            for (int w = 0; w < kOptBlock / 32; ++w) t2 += s_red[w];
            const float total_norm = (float)sqrt(t2);
            s_coef = fminf(max_norm / (total_norm + 1e-6f), 1.0f);
        }
    } else if (threadIdx.x == 0) {
        s_coef = 1.0f;
    }
    __syncthreads();
    const float coef = s_coef;
    const int t = blockIdx.y;
    const int64_t n = sizes[t];
    const double step = (double)*steps[t];
    const double bc1 = 1.0 - pow((double)beta1, step);
    const double bc2 = 1.0 - pow((double)beta2, step);
    const float step_size = (float)((lr_dev ? *lr_dev : (double)lr) / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
    float* __restrict__ p = params[t];
    const float* __restrict__ g = grads[t];
    float* __restrict__ m = exp_avg[t];
    float* __restrict__ v = exp_avg_sq[t];
    const float w1 = 1.0f - beta1, w2 = 1.0f - beta2;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float ge = g[e] * coef;
        const float me = m[e] + w1 * (ge - m[e]);
        const float ve = v[e] * beta2 + w2 * ge * ge;
        m[e] = me;
        v[e] = ve;
        const float denom = sqrtf(ve) / bc2_sqrt + eps;
        p[e] = p[e] - step_size * (me / denom);
    }
}

}  // namespace morl

extern "C" size_t morl_adam_workspace_bytes(int n_tensors, int64_t max_size) {
    long long bx = (max_size + morl::kOptBlock - 1) / morl::kOptBlock;
    if (bx > 64) bx = 64;
    if (bx < 1) bx = 1;
    return (size_t)n_tensors * (size_t)bx * sizeof(float);
}

static int adam_clip(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq, float* const* steps,
                     const int64_t* sizes, int n_tensors, int64_t max_size, float max_grad_norm, float lr, const double* lr_dev, float beta1,
                     float beta2, float eps, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(params && grads && exp_avg && exp_avg_sq && steps && sizes && workspace, MORL_ERR_NULL, "morl_adam_clip_f32: NULL pointer argument");
    MORL_REQUIRE(n_tensors > 0 && n_tensors <= 65535 && max_size > 0, MORL_ERR_SHAPE, "morl_adam_clip_f32: bad n_tensors=%d max_size=%lld", n_tensors,
                 (long long)max_size);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    long long bx = (max_size + kOptBlock - 1) / kOptBlock;
    if (bx > 64) bx = 64;
    const dim3 grid((unsigned)bx, (unsigned)n_tensors, 1);
    float* partials = static_cast<float*>(workspace);
    launch_k(grad_sqnorm_kernel, dim3(grid), dim3(kOptBlock), 0, st, grads, sizes, steps, partials);
    int rc = check_launch("morl_adam_clip_f32(norm)");
    if (rc) return rc;
    launch_k(adam_clip_kernel, dim3(grid), dim3(kOptBlock), 0, st, params, grads, exp_avg, exp_avg_sq, steps, sizes, partials, (int)(bx * n_tensors), max_grad_norm, lr, lr_dev,
                                                 beta1, beta2, eps);
    return check_launch("morl_adam_clip_f32");
}

extern "C" int morl_adam_clip_f32(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                                  float* const* steps, const int64_t* sizes, int n_tensors, int64_t max_size, float max_grad_norm, float lr,
                                  float beta1, float beta2, float eps, void* workspace, void* stream) {
    return adam_clip(params, grads, exp_avg, exp_avg_sq, steps, sizes, n_tensors, max_size, max_grad_norm, lr, nullptr, beta1, beta2, eps, workspace,
                     stream);
}

// The same update with the learning rate read from a device double at run time, so a captured graph follows a schedule (PPO's anneal_lr)
// without a re-capture.  A double keeps the Python float the reference's optimiser divides by its bias correction.
extern "C" int morl_adam_clip_lr_f32(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                                     float* const* steps, const int64_t* sizes, int n_tensors, int64_t max_size, float max_grad_norm,
                                     const double* lr, float beta1, float beta2, float eps, void* workspace, void* stream) {
    MORL_REQUIRE(lr, MORL_ERR_NULL, "morl_adam_clip_lr_f32: NULL learning rate");
    return adam_clip(params, grads, exp_avg, exp_avg_sq, steps, sizes, n_tensors, max_size, max_grad_norm, 0.f, lr, beta1, beta2, eps, workspace, stream);
}
