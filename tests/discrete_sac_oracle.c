/*
 * discrete_sac_oracle.c -- TEST INFRASTRUCTURE ONLY.  Plain-C restatement of the discrete-action MOSAC kernels of
 * morl_baselines_b200/csrc/discrete_sac.cu (reference single_policy/ser/mosac_discrete_action.py:452-498): the checker the kernels
 * equal bit for bit.  tests/discrete_sac_oracle.py compiles it on first use with
 *     cc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC
 * into a temporary directory; contraction is disabled so that every a*b+c below is two IEEE roundings unless fmaf() is written.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAP_TILE 0

/* w . q in MORL_DOT_UNFUSED (include/morl_b200.h): ((w0*q0 + w1*q1) + w2*q2) + ..., every operation rounded */
static float dotw(const float* w, const float* q, int D) {
    float acc = w[0] * q[0];
    for (int r = 1; r < D; ++r) {
        float p = w[r] * q[r];
        acc = acc + p;
    }
    return acc;
}

/* r + ((1 - done) * gamma) * q, three separate operations */
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


/* ---- discrete-action MOSAC, single_policy/ser/mosac_discrete_action.py:452-498 --------------------------------------------
 * The library's portable e^x and log x (csrc/discrete_sac.cu), restated operation for operation. */
static float f_from_bits(uint32_t b) {
    float f;
    memcpy(&f, &b, 4);
    return f;
}

static uint32_t bits_of(float f) {
    uint32_t b;
    memcpy(&b, &f, 4);
    return b;
}

float oracle_ds_exp(float x) {
    if (x != x) return x;
    if (x < -104.0f) return 0.0f;
    if (x > 89.0f) return f_from_bits(0x7f800000u);
    float j = rintf(x * 1.44269502f);
    float r = fmaf(j, -0.693145751953125f, x);
    r = fmaf(j, -1.42860677e-06f, r);
    float p = 1.98412698e-04f;
    p = fmaf(p, r, 1.38888889e-03f);
    p = fmaf(p, r, 8.33333333e-03f);
    p = fmaf(p, r, 4.16666667e-02f);
    p = fmaf(p, r, 1.66666667e-01f);
    p = fmaf(p, r, 0.5f);
    p = fmaf(p, r, 1.0f);
    p = fmaf(p, r, 1.0f);
    int ji = (int)j;
    int e1 = ji / 2, e2 = ji - e1;
    float a = p * f_from_bits((uint32_t)(e1 + 127) << 23);
    return a * f_from_bits((uint32_t)(e2 + 127) << 23);
}

float oracle_ds_log(float x) {
    if (x != x) return x;
    if (x < 0.0f) return f_from_bits(0x7fffffffu);
    if (x == 0.0f) return f_from_bits(0xff800000u);
    if (x == f_from_bits(0x7f800000u)) return x;
    int e = 0;
    if (x < 1.17549435e-38f) {
        x = x * 8388608.0f;
        e = -23;
    }
    uint32_t b = bits_of(x);
    e += (int)((b >> 23) & 255u) - 127;
    float m = f_from_bits((b & 0x007fffffu) | 0x3f800000u);
    if (m > 1.41421356f) {
        m = m * 0.5f;
        e += 1;
    }
    float f = m - 1.0f;
    float den = f + 2.0f;
    float u = f / den;
    float u2 = u * u;
    float q = fmaf(u2, 0.111111111f, 0.142857143f);
    q = fmaf(q, u2, 0.2f);
    q = fmaf(q, u2, 0.333333333f);
    float h = u + u;
    float hu2 = h * u2;
    float lm = fmaf(hu2, q, h);
    float ef = (float)e;
    return fmaf(ef, 0.693145751953125f, fmaf(ef, 1.42860677e-06f, lm));
}

/* th.min: NaN if either operand is NaN */
static float nan_min(float a, float b) {
    if (a != a || b != b) return f_from_bits(0x7fffffffu);
    return a < b ? a : b;
}

/* max (NaN propagates), sum_a e^(x - max) in action order, log of the sum */
static void ds_softmax_row(const float* x, int A, float* mx, float* s, float* lse) {
    float m = x[0];
    for (int a = 1; a < A; ++a)
        if (x[a] > m || x[a] != x[a]) m = x[a];
    float acc = 0.f;
    for (int a = 0; a < A; ++a) acc = acc + oracle_ds_exp(x[a] - m);
    *mx = m;
    *s = acc;
    *lse = oracle_ds_log(acc);
}

static float ds_critic_min(const float* q_nets, int n_nets, size_t stride, size_t off, const float* wv, int D) {
    float m = 0.f;
    for (int n = 0; n < n_nets; ++n) {
        float s = dotw(wv, q_nets + n * stride + off, D);
        m = (n == 0) ? s : nan_min(m, s);
    }
    return m;
}

/* :452-464  v = sum_a p (min_n w.q_n - alpha logp);  target = w.r + (1 - done) gamma v */
void oracle_discrete_sac_target(const float* q_nets, int n_nets, const float* logits, const float* w, int w_rows, int w_map,
                                const float* reward, const float* done, float alpha, float gamma, int N, int A, int D, float* out) {
    size_t stride = (size_t)N * A * D;
    for (int k = 0; k < N; ++k) {
        const float* wv = w + (size_t)map_row(k, w_rows, N, w_map) * D;
        const float* x = logits + (size_t)k * A;
        float mx, s, lse;
        ds_softmax_row(x, A, &mx, &s, &lse);
        float v = 0.f;
        for (int a = 0; a < A; ++a) {
            float z = x[a] - mx;
            float lp = z - lse;
            if (lp == -INFINITY) continue;
            float p = oracle_ds_exp(z) / s;
            float m = ds_critic_min(q_nets, n_nets, stride, ((size_t)k * A + a) * D, wv, D);
            float al = alpha * lp;
            float d = m - al;
            v = v + p * d;
        }
        float rs = dotw(wv, reward + (size_t)k * D, D);
        out[k] = bellman(rs, done[k], gamma, v);
    }
}

/* warp-shuffle butterfly of 32 lanes (v_l += v_{l^off}, off = 16 .. 1); the result of lane 0 */
static float warp_butterfly(float* v) {
    float t[32];
    for (int off = 16; off > 0; off >>= 1) {
        for (int l = 0; l < 32; ++l) t[l] = v[l] + v[l ^ off];
        memcpy(v, t, sizeof(t));
    }
    return v[0];
}

/* the kernel's block partial over 256 rows: per-warp butterflies, then warp 0 over the 8 warp sums */
static float block_partial_256(const float* rows, int n) {
    float red[32];
    for (int wp = 0; wp < 8; ++wp) {
        float v[32];
        for (int l = 0; l < 32; ++l) v[l] = (wp * 32 + l < n) ? rows[wp * 32 + l] : 0.f;
        red[wp] = warp_butterfly(v);
    }
    for (int l = 8; l < 32; ++l) red[l] = 0.f;
    return warp_butterfly(red);
}

/* 256 strided double accumulators over the block partials, then a halving tree */
static double final_sum_256(const float* partials, int n_blocks, int stride, int which) {
    double red[256];
    for (int t = 0; t < 256; ++t) {
        double a = 0.0;
        for (int b = t; b < n_blocks; b += 256) a += (double)partials[stride * b + which];
        red[t] = a;
    }
    for (int h = 128; h > 0; h >>= 1)
        for (int t = 0; t < h; ++t) red[t] += red[t + h];
    return red[0];
}

/* :478-498  actor loss mean(p (alpha logp - m)), its gradient p (f - sum_a p f) / (N A) w.r.t. the logits, and the temperature loss
 * mean(p (-e^log_alpha (logp + H))) with its derivative w.r.t. log_alpha; log_alpha NULL = no temperature outputs */
void oracle_discrete_sac_actor_loss(const float* logits, const float* q_nets, int n_nets, const float* w, int w_rows, int w_map, float alpha,
                                    const float* log_alpha, float target_entropy, int N, int A, int D, float* actor_loss, float* dlogits,
                                    float* alpha_loss, float* dlog_alpha) {
    if (N <= 0 || A <= 0) return;
    size_t stride = (size_t)N * A * D;
    int n_blocks = (N + 255) / 256;
    float* rows = (float*)malloc(sizeof(float) * 3 * (size_t)N);
    float* partials = (float*)calloc(3 * (size_t)n_blocks, sizeof(float));
    double inv_na = 1.0 / ((double)N * A);
    float inv_na_f = (float)inv_na;
    float t = log_alpha ? -oracle_ds_exp(log_alpha[0]) : 0.f;
    for (int k = 0; k < N; ++k) {
        const float* wv = w + (size_t)map_row(k, w_rows, N, w_map) * D;
        const float* x = logits + (size_t)k * A;
        float* g = dlogits ? dlogits + (size_t)k * A : NULL;
        float mx, s, lse;
        ds_softmax_row(x, A, &mx, &s, &lse);
        float l = 0.f, al = 0.f, c = 0.f;
        for (int a = 0; a < A; ++a) {
            float z = x[a] - mx;
            float lp = z - lse;
            if (lp == -INFINITY) continue;
            float p = oracle_ds_exp(z) / s;
            float m = ds_critic_min(q_nets, n_nets, stride, ((size_t)k * A + a) * D, wv, D);
            float f = alpha * lp;
            f = f - m;
            float pf = p * f;
            l = l + pf;
            if (log_alpha) {
                float u = lp + target_entropy;
                float pu = p * u;
                c = c + pu;
                float tu = t * u;
                float ptu = p * tu;
                al = al + ptu;
            }
            if (g) g[a] = f;
        }
        if (g) {
            for (int a = 0; a < A; ++a) {
                float z = x[a] - mx;
                float lp = z - lse;
                float v = 0.f;
                if (lp != -INFINITY) {
                    float p = oracle_ds_exp(z) / s;
                    float d = g[a] - l;
                    float pd = p * d;
                    v = pd * inv_na_f;
                }
                g[a] = v;
            }
        }
        rows[k] = l;
        rows[N + k] = al;
        rows[2 * (size_t)N + k] = c;
    }
    for (int b = 0; b < n_blocks; ++b) {
        int n = (N - b * 256) < 256 ? (N - b * 256) : 256;
        for (int i = 0; i < 3; ++i) partials[3 * b + i] = block_partial_256(rows + (size_t)i * N + (size_t)b * 256, n);
    }
    actor_loss[0] = (float)(final_sum_256(partials, n_blocks, 3, 0) * inv_na);
    if (log_alpha) {
        alpha_loss[0] = (float)(final_sum_256(partials, n_blocks, 3, 1) * inv_na);
        dlog_alpha[0] = (float)((double)t * final_sum_256(partials, n_blocks, 3, 2) * inv_na);
    }
    free(rows);
    free(partials);
}
