// replay.cu -- device-resident replay store: minibatch index gather (SURVEY.md K8) and the PER sum-tree (K9).
//
// Replaces ReplayBuffer.sample's five fancy-index gathers + six host->device copies (reference common/buffer.py:82-94,
// common/prioritized_buffer.py:160-166) with one kernel over stores that already live in HBM, and SumTree.sample /
// SumTree.batch_set (common/prioritized_buffer.py:30-54, 69-82) with device kernels over the same float64 level arrays.
#include "common.cuh"

namespace morl {

__device__ __forceinline__ int64_t clamp_idx(int64_t v, int64_t cap) { return v < 0 ? 0 : (v >= cap ? cap - 1 : v); }

// One launch gathers all five arrays.  obs / next_obs rows are moved as 128-bit words when obs_dim % 4 == 0.
template <bool VEC4>
__global__ void __launch_bounds__(256) replay_gather_kernel(const float* __restrict__ obs_store, const float* __restrict__ next_obs_store,
                                                            const void* __restrict__ act_store, const float* __restrict__ rew_store,
                                                            const float* __restrict__ done_store, const int64_t* __restrict__ idx, int B,
                                                            int obs_dim, int act_dim, int rew_dim, int act_is_u8, int64_t capacity,
                                                            float* __restrict__ obs_out, float* __restrict__ next_obs_out,
                                                            void* __restrict__ act_out, float* __restrict__ rew_out,
                                                            float* __restrict__ done_out) {
    pdl_enter();
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    if constexpr (VEC4) {
        const int vpr = obs_dim / 4;  // float4 per row
        const long long total = (long long)B * vpr;
        const float4* o4 = reinterpret_cast<const float4*>(obs_store);
        const float4* n4 = reinterpret_cast<const float4*>(next_obs_store);
        float4* oo = reinterpret_cast<float4*>(obs_out);
        float4* no = reinterpret_cast<float4*>(next_obs_out);
        for (long long e = tid; e < total; e += nthreads) {
            const int row = (int)(e / vpr);
            const int c = (int)(e - (long long)row * vpr);
            const int64_t src = clamp_idx(__ldg(idx + row), capacity) * vpr + c;
            oo[e] = __ldg(o4 + src);
            no[e] = __ldg(n4 + src);
        }
    } else {
        const long long total = (long long)B * obs_dim;
        for (long long e = tid; e < total; e += nthreads) {
            const int row = (int)(e / obs_dim);
            const int c = (int)(e - (long long)row * obs_dim);
            const int64_t src = clamp_idx(__ldg(idx + row), capacity) * obs_dim + c;
            obs_out[e] = __ldg(obs_store + src);
            next_obs_out[e] = __ldg(next_obs_store + src);
        }
    }
    for (long long e = tid; e < (long long)B * rew_dim; e += nthreads) {
        const int row = (int)(e / rew_dim);
        const int c = (int)(e - (long long)row * rew_dim);
        rew_out[e] = __ldg(rew_store + clamp_idx(__ldg(idx + row), capacity) * rew_dim + c);
    }
    for (long long e = tid; e < (long long)B * act_dim; e += nthreads) {
        const int row = (int)(e / act_dim);
        const int c = (int)(e - (long long)row * act_dim);
        const int64_t src = clamp_idx(__ldg(idx + row), capacity) * act_dim + c;
        if (act_is_u8)
            static_cast<int32_t*>(act_out)[e] = (int32_t) static_cast<const uint8_t*>(act_store)[src];
        else
            static_cast<float*>(act_out)[e] = static_cast<const float*>(act_store)[src];
    }
    for (long long e = tid; e < B; e += nthreads) done_out[e] = __ldg(done_store + clamp_idx(__ldg(idx + e), capacity));
}

}  // namespace morl

extern "C" int morl_replay_gather(const float* obs_store, const float* next_obs_store, const void* act_store, const float* rew_store,
                                  const float* done_store, const int64_t* idx, int B, int obs_dim, int act_dim, int rew_dim,
                                  int act_is_u8, int64_t capacity, float* obs_out, float* next_obs_out, void* act_out,
                                  float* rew_out, float* done_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(obs_store && next_obs_store && act_store && rew_store && done_store && idx && obs_out && next_obs_out && act_out &&
                     rew_out && done_out,
                 MORL_ERR_NULL, "morl_replay_gather: NULL pointer argument");
    MORL_REQUIRE(B > 0 && obs_dim > 0 && act_dim > 0 && rew_dim > 0 && capacity > 0, MORL_ERR_SHAPE,
                 "morl_replay_gather: bad shape B=%d obs_dim=%d act_dim=%d rew_dim=%d capacity=%lld", B, obs_dim, act_dim, rew_dim,
                 (long long)capacity);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec4 = (obs_dim % 4 == 0) && aligned16(obs_store) && aligned16(next_obs_store) && aligned16(obs_out) && aligned16(next_obs_out);
    const long long work = (long long)B * (vec4 ? obs_dim / 4 : obs_dim);
    long long blocks = (work + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (vec4)
        launch_k(replay_gather_kernel<true>, dim3((int)blocks), dim3(256), 0, st, obs_store, next_obs_store, act_store, rew_store, done_store, idx, B, obs_dim,
                                                                act_dim, rew_dim, act_is_u8, capacity, obs_out, next_obs_out, act_out,
                                                                rew_out, done_out);
    else
        launch_k(replay_gather_kernel<false>, dim3((int)blocks), dim3(256), 0, st, obs_store, next_obs_store, act_store, rew_store, done_store, idx, B, obs_dim,
                                                                 act_dim, rew_dim, act_is_u8, capacity, obs_out, next_obs_out, act_out,
                                                                 rew_out, done_out);
    return check_launch("morl_replay_gather");
}
