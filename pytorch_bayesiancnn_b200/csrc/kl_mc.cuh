// Monte-Carlo KL against the scale-mixture prior of Bayes by Backprop (Blundell et al. 2015, section 3.3),
//   p(w) = pi N(w; 0, sigma1^2) + (1 - pi) N(w; 0, sigma2^2),
// which has no closed form.  For q = N(mu, sigma^2), sigma = log1p(exp(rho)), and one standard normal eps per element:
//   w    = mu + sigma eps
//   term = -log sigma - 1/2 - logsumexp(log pi - log sigma1 - w^2 / (2 sigma1^2), log(1 - pi) - log sigma2 - w^2 / (2 sigma2^2))
// The entropy half is analytic, only the cross-entropy half is sampled; the two 1/2 log 2 pi cancel.  Always an estimate
// of KL(q || p): kl_convention does not apply.
// Element i of W draws normal(i) of the draw's Philox stream, bias element n draws normal(|W| + n); draw d of a call uses
// stream + d * stride, so the draws of folded Monte-Carlo samples are those of one call per sample.
#pragma once
#include "common.cuh"

namespace bbb {

// The two logsumexp arguments of weight w are lc[k] - w^2 h[k]:  lc = log(weight_k / sigma_k), h = 1 / (2 sigma_k^2).
// pi = 1: lc[1] = -inf, and the spike drops out of the max-subtracted logsumexp.
struct MixPrior { float lc1, lc2, h1, h2; };

constexpr int KL_MC_THREADS = 256;
constexpr int KL_MC_MAX_DRAWS = 16;      // draws of one launch: a double accumulator per thread and draw in shared memory

// -log p(w) up to the constant; with r2 (nullable) the spike's responsibility, softmax of the two arguments.
// Max-subtracted, so it stays finite when w^2 h2 overflows (b = -inf): the slab's exponent does not.
__device__ __forceinline__ float mix_neg_log_p(float w, const MixPrior& q, float* r2) {
    const float w2 = w * w;
    const float a = q.lc1 - w2 * q.h1, b = q.lc2 - w2 * q.h2;
    const float e = expf(-fabsf(a - b));                 // a finite: |a - b| is never NaN
    const float lse = fmaxf(a, b) + log1pf(e);
    if (r2) { const float lo = e / (1.0f + e); *r2 = b > a ? 1.0f - lo : lo; }
    return -lse;
}

struct Mu4 { float v[4]; };
__device__ __forceinline__ Mu4 load4(const float* __restrict__ p, uint64_t grp, bool vec) {
    Mu4 o;
    if (vec) { const float4 t = __ldg(reinterpret_cast<const float4*>(p) + grp); o.v[0] = t.x; o.v[1] = t.y; o.v[2] = t.z; o.v[3] = t.w; }
    else {
#pragma unroll
        for (int j = 0; j < 4; ++j) o.v[j] = __ldg(p + 4 * grp + j);
    }
    return o;
}

// n_draws (<= KL_MC_MAX_DRAWS) sums, kl_out[d] from stream + d * stride.  mu and rho are read once; work item t is the
// four weights 4t .. 4t+3 (one normal4 per draw) for t < n_w / 4, then one by one the n_w % 4 last weights and the bias.
// Every draw accumulates the same items in the same order, in double, and finishes through kl_publish with a counter and
// a partial row of its own (workspace: counters[n_draws], padded to 256 bytes, then partials[n_draws][gridDim.x]).
__global__ void __launch_bounds__(KL_MC_THREADS)
kl_mc_forward_kernel(const float* __restrict__ w_mu, const float* __restrict__ w_rho, uint64_t n_w,
                     const float* __restrict__ b_mu, const float* __restrict__ b_rho, uint64_t n_b, MixPrior q,
                     NoiseKey key, const unsigned long long* stream_base, int n_draws, unsigned long long stride,
                     unsigned int* counters, double* partials, float* kl_out) {
    extern __shared__ double mc_acc[];               // [n_draws][KL_MC_THREADS]
    __shared__ double red[32];
    const McFold draws{0, 0, stride, 1, 0};
    const NoiseKey k0 = effective_key(key, stream_base);
    for (int d = 0; d < n_draws; ++d) mc_acc[d * KL_MC_THREADS + threadIdx.x] = 0.0;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
    const bool vec = ((((uintptr_t)w_mu) | ((uintptr_t)w_rho)) & 15u) == 0;
    const uint64_t n4 = n_w >> 2;
    for (uint64_t g = tid; g < n4; g += nth) {
        const Mu4 m = load4(w_mu, g, vec), r = load4(w_rho, g, vec);
        float sg[4], ent = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; ++j) { sg[j] = softplus_sigma(r.v[j]); ent += -logf(sg[j]) - 0.5f; }
        for (int d = 0; d < n_draws; ++d) {
            const float4 z = normal4(g, sample_key(k0, draws, d));
            const float e[4] = {z.x, z.y, z.z, z.w};
            float s = ent;
#pragma unroll
            for (int j = 0; j < 4; ++j) s += mix_neg_log_p(fmaf(sg[j], e[j], m.v[j]), q, nullptr);
            mc_acc[d * KL_MC_THREADS + threadIdx.x] += (double)s;
        }
    }
    const uint64_t tail0 = n4 << 2, n_tail = (n_w - tail0) + n_b;
    for (uint64_t t = tid; t < n_tail; t += nth) {
        const uint64_t i = tail0 + t;                    // the element's draw index: |W| + n for bias element n
        const bool bias = i >= n_w;
        const float m = bias ? __ldg(b_mu + (i - n_w)) : __ldg(w_mu + i);
        const float sg = softplus_sigma(bias ? __ldg(b_rho + (i - n_w)) : __ldg(w_rho + i));
        const float ent = -logf(sg) - 0.5f;
        for (int d = 0; d < n_draws; ++d) {
            const float e = normal1(i, sample_key(k0, draws, d));
            mc_acc[d * KL_MC_THREADS + threadIdx.x] += (double)(ent + mix_neg_log_p(fmaf(sg, e, m), q, nullptr));
        }
    }
    for (int d = 0; d < n_draws; ++d) {
        const double tot = block_sum(mc_acc[d * KL_MC_THREADS + threadIdx.x], red);
        if (threadIdx.x == 0) kl_publish(tot, blockIdx.x, gridDim.x, partials + (size_t)d * gridDim.x, counters + d, kl_out + d);
        __syncthreads();                                 // `red` is reused by the next draw
    }
}

// Reparameterisation gradients of the n elements (mu, rho), which drew normal(first + i):
//   s = w (r1 / sigma1^2 + r2 / sigma2^2) = -d log p / dw ;  d/dmu = s ;  d/dsigma = -1/sigma + s eps ;  d/drho = sigmoid(rho) d/dsigma
// g_mu / g_rho += sum_d grad_kl[d] * (...), draws in ascending order.  Groups of four elements share a normal4 when the
// first draw index is a multiple of four (a weight tensor); otherwise (a bias behind |W| % 4 != 0 weights) one by one.
__device__ __forceinline__ void kl_mc_grad_elem(float m, float sg, float sig, float e, float go, const MixPrior& q,
                                                float& gm, float& gr) {
    float r2;
    const float w = fmaf(sg, e, m);
    mix_neg_log_p(w, q, &r2);
    const float s = w * (2.0f * q.h1 * (1.0f - r2) + 2.0f * q.h2 * r2);
    gm += go * s;
    gr += go * (s * e - 1.0f / sg) * sig;
}

__global__ void __launch_bounds__(KL_MC_THREADS)
kl_mc_backward_kernel(const float* __restrict__ mu, const float* __restrict__ rho, uint64_t n, uint64_t first, MixPrior q,
                      NoiseKey key, const unsigned long long* stream_base, int n_draws, unsigned long long stride,
                      const float* __restrict__ grad_kl, float* __restrict__ g_mu, float* __restrict__ g_rho) {
    const McFold draws{0, 0, stride, 1, 0};
    const NoiseKey k0 = effective_key(key, stream_base);
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
    const bool vec = ((((uintptr_t)mu) | ((uintptr_t)rho) | ((uintptr_t)g_mu) | ((uintptr_t)g_rho)) & 15u) == 0;
    const uint64_t n4 = (first & 3u) == 0 ? (n >> 2) : 0;
    for (uint64_t g = tid; g < n4; g += nth) {
        const Mu4 m = load4(mu, g, vec), r = load4(rho, g, vec);
        float sg[4], sig[4], gm[4] = {0.0f, 0.0f, 0.0f, 0.0f}, gr[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int j = 0; j < 4; ++j) { sg[j] = softplus_sigma(r.v[j]); sig[j] = 1.0f / (1.0f + expf(-r.v[j])); }
        for (int d = 0; d < n_draws; ++d) {
            const float go = __ldg(grad_kl + d);
            const float4 z = normal4((first >> 2) + g, sample_key(k0, draws, d));
            const float e[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) kl_mc_grad_elem(m.v[j], sg[j], sig[j], e[j], go, q, gm[j], gr[j]);
        }
        if (vec) {
            float4* pm = reinterpret_cast<float4*>(g_mu) + g; float4* pr = reinterpret_cast<float4*>(g_rho) + g;
            const float4 am = *pm, ar = *pr;
            *pm = make_float4(am.x + gm[0], am.y + gm[1], am.z + gm[2], am.w + gm[3]);
            *pr = make_float4(ar.x + gr[0], ar.y + gr[1], ar.z + gr[2], ar.w + gr[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) { g_mu[4 * g + j] += gm[j]; g_rho[4 * g + j] += gr[j]; }
        }
    }
    for (uint64_t i = (n4 << 2) + tid; i < n; i += nth) {
        const float m = __ldg(mu + i), r = __ldg(rho + i);
        const float sg = softplus_sigma(r), sig = 1.0f / (1.0f + expf(-r));
        float gm = 0.0f, gr = 0.0f;
        for (int d = 0; d < n_draws; ++d)
            kl_mc_grad_elem(m, sg, sig, normal1(first + i, sample_key(k0, draws, d)), __ldg(grad_kl + d), q, gm, gr);
        g_mu[i] += gm;
        g_rho[i] += gr;
    }
}

}  // namespace bbb
