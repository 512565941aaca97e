// pair_layer1.cu -- the separable first layer of the weight-conditioned Q-network on the pair batch: both input products in one small
// launch instead of two library sgemms and their epilogue kernels.
//
// Reference: QNet.forward builds [s || w] rows and runs nn.Linear on B*W (reference: B*W^2) of them
// (multi_policy/envelope/envelope.py:59-77).  Here  W1 [s || w] + b1 = W1_s s + (W1_w w + b1)  (DESIGN.md section 2), so only
//     u[b, :] = W1_s feats[b]                 (B rows, K = F)
//     v[j, :] = W1_w wset[j] + b1            (W rows, K = D)
// are computed (morl_pair_layer1_uv_f32: 6.3 us; the library path was two SIMT sgemms plus their epilogue kernels, ~15 us).  The
// parameter gradients dW1 = [dU^T feats | dV^T wset], db1 = colsum(dV) are ONE launch as well (morl_pair_layer1_grad_f32: split
// reduction over the transitions, partial tiles summed in a fixed order by the last block of each column tile), replacing two library
// sgemms + split-K reduce + cat + sum of the round-1 path.
// fp32 FMA chains in a fixed order: deterministic, and within the 1e-5 parity bar of the dense layers (tests/test_gemm_gpu.py).
#include "common.cuh"

namespace morl {

constexpr int kL1Rows = 8;  // rows (transitions or weight vectors) per block of the forward kernel

// grid.x = ceil((B + W) / kL1Rows), block = 256 threads striding the H outputs.  W1 is row-major [H, F + D].
__global__ void __launch_bounds__(256) pair_layer1_uv_kernel(const float* __restrict__ feats, const float* __restrict__ wset, const float* __restrict__ W1,
                                                             const float* __restrict__ b1, int B, int W, int F, int D, int H, float* __restrict__ u,
                                                             float* __restrict__ v) {
    pdl_enter();
    extern __shared__ float xs[];  // [kL1Rows][max(F, D)] input rows of this block
    const int K = F + D;
    const int r0 = blockIdx.x * kL1Rows;
    const int kmax = F > D ? F : D;
    for (int t = threadIdx.x; t < kL1Rows * kmax; t += blockDim.x) {
        const int rr = t / kmax, k = t - rr * kmax;
        const int r = r0 + rr;
        float x = 0.f;
        if (r < B) {
            if (k < F) x = __ldg(feats + (size_t)r * F + k);
        } else if (r < B + W) {
            if (k < D) x = __ldg(wset + (size_t)(r - B) * D + k);
        }
        xs[t] = x;
    }
    __syncthreads();
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
        const float* wrow = W1 + (size_t)h * K;
        float accu[kL1Rows];
#pragma unroll
        for (int rr = 0; rr < kL1Rows; ++rr) accu[rr] = 0.f;
        // rows of this block are either all transitions, all weight vectors, or (one block at most) mixed: handle per row
        const bool any_u = r0 < B, any_v = r0 + kL1Rows > B;
        if (any_u) {
            for (int k = 0; k < F; ++k) {
                const float wk = __ldg(wrow + k);
#pragma unroll
                for (int rr = 0; rr < kL1Rows; ++rr)
                    if (r0 + rr < B) accu[rr] = __fmaf_rn(xs[rr * kmax + k], wk, accu[rr]);
            }
        }
        if (any_v) {
            const float bias = __ldg(b1 + h);
#pragma unroll
            for (int rr = 0; rr < kL1Rows; ++rr)
                if (r0 + rr >= B) accu[rr] = bias;
            for (int k = 0; k < D; ++k) {
                const float wk = __ldg(wrow + F + k);
#pragma unroll
                for (int rr = 0; rr < kL1Rows; ++rr)
                    if (r0 + rr >= B) accu[rr] = __fmaf_rn(xs[rr * kmax + k], wk, accu[rr]);
            }
        }
#pragma unroll
        for (int rr = 0; rr < kL1Rows; ++rr) {
            const int r = r0 + rr;
            if (r < B)
                u[(size_t)r * H + h] = accu[rr];
            else if (r < B + W)
                v[(size_t)(r - B) * H + h] = accu[rr];
        }
    }
}

// ---- product-conditioned first layer (GPI-PD's QNet): u = relu(s Ls^T + bs) on the B observations, v = relu(m Lw^T + bw) on the P weight
// vectors, in one launch; grid.x = ceil((B + P) / kL1Rows), rows < B are observations.  Ls [H, F], Lw [H, D] row-major (nn.Linear).
__global__ void __launch_bounds__(256) product_layer1_uv_kernel(const float* __restrict__ s, const float* __restrict__ Ls, const float* __restrict__ bs,
                                                                const float* __restrict__ m, const float* __restrict__ Lw, const float* __restrict__ bw,
                                                                int B, int P, int F, int D, int H, float* __restrict__ u, float* __restrict__ v) {
    pdl_enter();
    extern __shared__ float xs[];  // [kL1Rows][max(F, D)]
    const int r0 = blockIdx.x * kL1Rows;
    const int kmax = F > D ? F : D;
    for (int t = threadIdx.x; t < kL1Rows * kmax; t += blockDim.x) {
        const int rr = t / kmax, k = t - rr * kmax;
        const int r = r0 + rr;
        float x = 0.f;
        if (r < B) {
            if (k < F) x = __ldg(s + (size_t)r * F + k);
        } else if (r < B + P) {
            if (k < D) x = __ldg(m + (size_t)(r - B) * D + k);
        }
        xs[t] = x;
    }
    __syncthreads();
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
        float accu[kL1Rows];
        const float b_s = __ldg(bs + h), b_w = __ldg(bw + h);
#pragma unroll
        for (int rr = 0; rr < kL1Rows; ++rr) accu[rr] = r0 + rr < B ? b_s : b_w;
        if (r0 < B) {
            for (int k = 0; k < F; ++k) {
                const float wk = __ldg(Ls + (size_t)h * F + k);
#pragma unroll
                for (int rr = 0; rr < kL1Rows; ++rr)
                    if (r0 + rr < B) accu[rr] = __fmaf_rn(xs[rr * kmax + k], wk, accu[rr]);
            }
        }
        if (r0 + kL1Rows > B) {
            for (int k = 0; k < D; ++k) {
                const float wk = __ldg(Lw + (size_t)h * D + k);
#pragma unroll
                for (int rr = 0; rr < kL1Rows; ++rr)
                    if (r0 + rr >= B) accu[rr] = __fmaf_rn(xs[rr * kmax + k], wk, accu[rr]);
            }
        }
#pragma unroll
        for (int rr = 0; rr < kL1Rows; ++rr) {
            const int r = r0 + rr;
            const float y = accu[rr] <= 0.f ? 0.f : accu[rr];  // ReLU (-0 -> +0, NaN propagates)
            if (r < B)
                u[(size_t)r * H + h] = y;
            else if (r < B + P)
                v[(size_t)(r - B) * H + h] = y;
        }
    }
}

// ---- backward: dW1 [H, F + D] = [dU^T feats | dV^T wset], db1 [H] = colsum(dV) -------------------------------------------------------------
// grid = (ceil(H / 32), kL1Splits); block 256 = 32 output rows h (lane) x 8 column groups (warp).  Split s reduces transitions
// [s*bs, (s+1)*bs) into the F "u" columns and weight vectors [s*js, (s+1)*js) into the D "v" columns + the bias column.  A chunk of
// reduction rows is staged ONCE in shared memory and every thread accumulates all of its columns (c = warp, warp + 8, ...) from it in
// registers; the partial tiles go to workspace[s][H][F + D + 1] and the LAST block of an h-tile to finish (self-resetting arrival counter)
// adds the kL1Splits partials in split order: deterministic, no float atomics.
constexpr int kL1Splits = 16;
constexpr int kL1Chunk = 32;   // reduction rows staged per pass
constexpr int kL1ColsPerThread = 8;  // columns per thread per column block (8 groups x 8 = 64 columns per block of columns)

__global__ void __launch_bounds__(256) pair_layer1_grad_kernel(const float* __restrict__ dU, const float* __restrict__ dV, const float* __restrict__ feats,
                                                               const float* __restrict__ wset, int B, int W, int F, int D, int H, float* __restrict__ dW1,
                                                               float* __restrict__ db1, float* __restrict__ partial, unsigned int* __restrict__ counters) {
    pdl_enter();
    __shared__ float gs[kL1Chunk][33];                          // gradient rows (dU or dV) of the chunk, this block's 32 h columns
    __shared__ float xs[kL1Chunk][8 * kL1ColsPerThread + 1];    // input rows of the chunk, the current block of <= 64 columns
    __shared__ unsigned int s_last;
    const int C = F + D + 1;
    const int h0 = blockIdx.x * 32, s = blockIdx.y;
    const int hl = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int bs = (B + kL1Splits - 1) / kL1Splits, js = (W + kL1Splits - 1) / kL1Splits;
    for (int cb = 0; cb < C; cb += 8 * kL1ColsPerThread) {  // column blocks of 64 (one for the usual F + D + 1 <= 64)
        const int ncol = min(8 * kL1ColsPerThread, C - cb);
        float acc[kL1ColsPerThread];
#pragma unroll
        for (int k = 0; k < kL1ColsPerThread; ++k) acc[k] = 0.f;
        for (int phase = 0; phase < 2; ++phase) {  // 0: transitions (u columns [0, F)), 1: weight vectors (v columns [F, F + D) + bias column)
            const int lo = phase == 0 ? s * bs : s * js, hi = phase == 0 ? min(B, lo + bs) : min(W, lo + js);
            const int c_lo = phase == 0 ? 0 : F, c_hi = phase == 0 ? F : C;   // global column range this phase contributes to
            if (cb >= c_hi || cb + ncol <= c_lo) continue;                   // (uniform) nothing of this column block in this phase
            const float* g = phase == 0 ? dU : dV;
            for (int r0 = lo; r0 < hi; r0 += kL1Chunk) {
                const int nr = min(kL1Chunk, hi - r0);
                __syncthreads();
                for (int t = threadIdx.x; t < nr * 32; t += 256) {
                    const int rr = t >> 5, hh = t & 31;
                    gs[rr][hh] = (h0 + hh < H) ? __ldg(g + (size_t)(r0 + rr) * H + h0 + hh) : 0.f;
                }
                for (int t = threadIdx.x; t < nr * 64; t += 256) {
                    const int rr = t >> 6, cl = t & 63, c = cb + cl;
                    float x = 0.f;  // columns of the other phase (and beyond the last column) contribute nothing here
                    if (cl >= ncol) {
                    } else if (phase == 0) {
                        if (c < F) x = __ldg(feats + (size_t)(r0 + rr) * F + c);
                    } else {
                        if (c >= F && c < F + D) x = __ldg(wset + (size_t)(r0 + rr) * D + (c - F));
                        else if (c == F + D) x = 1.0f;  // bias column: plain column sum of dV
                    }
                    xs[rr][cl] = x;
                }
                __syncthreads();
                for (int rr = 0; rr < nr; ++rr) {
                    const float gv = gs[rr][hl];
#pragma unroll
                    for (int k = 0; k < kL1ColsPerThread; ++k) acc[k] = __fmaf_rn(gv, xs[rr][grp + 8 * k], acc[k]);
                }
            }
        }
        if (h0 + hl < H) {
#pragma unroll
            for (int k = 0; k < kL1ColsPerThread; ++k) {
                const int c = cb + grp + 8 * k;
                if (grp + 8 * k < ncol) partial[((size_t)s * H + h0 + hl) * C + c] = acc[k];
            }
        }
    }
    // ---- last block of this h-tile sums the partial tiles in split order
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(counters + blockIdx.x, 1u);
        s_last = (prev == (unsigned int)(kL1Splits - 1));
        if (s_last) counters[blockIdx.x] = 0u;  // self-resetting: the workspace needs zeroing only once
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (h0 + hl >= H) return;
    // every partial of up to kL1TailCols columns of this thread is loaded FIRST (independent loads in flight together: one L2 latency
    // for the whole tail instead of one per column and split), then summed in four interleaved chains in split order (deterministic)
    constexpr int kL1TailCols = 5;  // 8 groups x 5 = 40 columns per pass (F + D + 1 = 36 at the north-star shape)
    for (int cb = grp; cb < C; cb += 8 * kL1TailCols) {
        float v[kL1TailCols][kL1Splits];
#pragma unroll
        for (int i = 0; i < kL1TailCols; ++i) {
            const int c = cb + 8 * i;
#pragma unroll
            for (int ss = 0; ss < kL1Splits; ++ss) v[i][ss] = c < C ? __ldcg(partial + ((size_t)ss * H + h0 + hl) * C + c) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < kL1TailCols; ++i) {
            const int c = cb + 8 * i;
            if (c >= C) break;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
            for (int ss = 0; ss < kL1Splits; ss += 4) {
                a0 += v[i][ss];
                a1 += v[i][ss + 1];
                a2 += v[i][ss + 2];
                a3 += v[i][ss + 3];
            }
            const float acc = (a0 + a1) + (a2 + a3);
            if (c < F + D)
                dW1[(size_t)(h0 + hl) * (F + D) + c] = acc;
            else
                db1[h0 + hl] = acc;
        }
    }
}

}  // namespace morl

extern "C" int morl_pair_layer1_uv_f32(const float* feats, const float* wset, const float* W1, const float* b1, int B, int W, int F, int D, int H, float* u,
                                       float* v, void* stream) {
    using namespace morl;
    MORL_REQUIRE(feats && wset && W1 && b1 && u && v, MORL_ERR_NULL, "morl_pair_layer1_uv_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && F > 0 && D > 0 && H > 0, MORL_ERR_SHAPE, "morl_pair_layer1_uv_f32: bad shape B=%d W=%d F=%d D=%d H=%d", B, W, F, D, H);
    const int kmax = F > D ? F : D;
    const size_t smem = (size_t)kL1Rows * kmax * sizeof(float);
    MORL_REQUIRE(smem <= 48 * 1024, MORL_ERR_UNSUPPORTED, "morl_pair_layer1_uv_f32: feature dimension %d too large", kmax);
    const int blocks = (B + W + kL1Rows - 1) / kL1Rows;
    launch_k(pair_layer1_uv_kernel, dim3(blocks), dim3(256), smem, static_cast<cudaStream_t>(stream), feats, wset, W1, b1, B, W, F, D, H, u, v);
    return check_launch("morl_pair_layer1_uv_f32");
}

extern "C" size_t morl_pair_layer1_grad_workspace_bytes(int F, int D, int H) {
    using namespace morl;
    if (F <= 0 || D <= 0 || H <= 0) return 0;
    // [kL1Splits][H][F + D + 1] fp32 partial tiles + one arrival counter per 32-row tile (the counters must be ZERO before the first call)
    return ((size_t)kL1Splits * H * (F + D + 1) + (size_t)(H + 31) / 32 + 4) * sizeof(float);
}

extern "C" int morl_pair_layer1_grad_f32(const float* dU, const float* dV, const float* feats, const float* wset, int B, int W, int F, int D, int H,
                                         float* dW1, float* db1, void* workspace, void* stream) {
    using namespace morl;
    MORL_REQUIRE(dU && dV && feats && wset && dW1 && db1 && workspace, MORL_ERR_NULL, "morl_pair_layer1_grad_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && F > 0 && D > 0 && H > 0, MORL_ERR_SHAPE, "morl_pair_layer1_grad_f32: bad shape B=%d W=%d F=%d D=%d H=%d", B, W, F, D, H);
    float* partial = static_cast<float*>(workspace);
    unsigned int* counters = reinterpret_cast<unsigned int*>(partial + (size_t)kL1Splits * H * (F + D + 1));
    dim3 grid((H + 31) / 32, kL1Splits);
    launch_k(pair_layer1_grad_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), dU, dV, feats, wset, B, W, F, D, H, dW1, db1, partial, counters);
    return check_launch("morl_pair_layer1_grad_f32");
}

extern "C" int morl_product_layer1_uv_f32(const float* s, const float* Ls, const float* bs, int B, int F, const float* m, const float* Lw, const float* bw,
                                          int P, int D, int H, float* u, float* v, void* stream) {
    using namespace morl;
    MORL_REQUIRE(s && Ls && bs && m && Lw && bw && u && v, MORL_ERR_NULL, "morl_product_layer1_uv_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && P > 0 && F > 0 && D > 0 && H > 0, MORL_ERR_SHAPE, "morl_product_layer1_uv_f32: bad shape B=%d P=%d F=%d D=%d H=%d", B, P, F, D, H);
    const int kmax = F > D ? F : D;
    const size_t smem = (size_t)kL1Rows * kmax * sizeof(float);
    MORL_REQUIRE(smem <= 48 * 1024, MORL_ERR_UNSUPPORTED, "morl_product_layer1_uv_f32: input dimension %d too large", kmax);
    const int blocks = (B + P + kL1Rows - 1) / kL1Rows;
    launch_k(product_layer1_uv_kernel, dim3(blocks), dim3(256), smem, static_cast<cudaStream_t>(stream), s, Ls, bs, m, Lw, bw, B, P, F, D, H, u, v);
    return check_launch("morl_product_layer1_uv_f32");
}
