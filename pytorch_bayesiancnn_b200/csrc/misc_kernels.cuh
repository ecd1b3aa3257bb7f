// Stand-alone KL forward/backward, Philox fill and the Monte-Carlo combine.
#pragma once
#include "common.cuh"

namespace bbb {

// kl_loss() without a preceding forward (SURVEY.md D7): sigma recomputed from rho.
// HBM-bound: reads 8 B per weight once (16 B with a tensor prior), float4-vectorised when aligned.
// TP: the prior of element i is (q.w_mu[i], q.w_sigma[i]) / (q.b_mu[i], q.b_sigma[i]) (bbb_prior) instead of (pm, ps);
// same loops, so the same summation order.  MK: a pruned element (q.w_mask / q.b_mask) adds +0.0 in its own place.
template <bool TP, bool MK = false>
__device__ __forceinline__ void kl_forward_body(const float* __restrict__ w_mu, const float* __restrict__ w_rho, uint64_t n_w,
                                                const float* __restrict__ b_mu, const float* __restrict__ b_rho, uint64_t n_b,
                                                float pm, float ps, const PriorPtrs& q, int conv, double* partials,
                                                unsigned int* counter, float* kl_out) {
    __shared__ double red[32];
    double acc = 0.0;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
    uintptr_t align = ((uintptr_t)w_mu) | ((uintptr_t)w_rho);
    if (TP) align |= ((uintptr_t)q.w_mu) | ((uintptr_t)q.w_sigma);
    const bool vec = (align & 15u) == 0;
    const uint64_t n4 = vec ? (n_w >> 2) : 0;
    for (uint64_t i = tid; i < n4; i += nth) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(w_mu) + i);
        const float4 r = __ldg(reinterpret_cast<const float4*>(w_rho) + i);
        float4 a = make_float4(pm, pm, pm, pm), b = make_float4(ps, ps, ps, ps);
        if (TP) { a = __ldg(reinterpret_cast<const float4*>(q.w_mu) + i); b = __ldg(reinterpret_cast<const float4*>(q.w_sigma) + i); }
        const auto w_in = [&](int j) { return kept(w_keep<MK>(q, 4 * i + j)); };
        float s = w_in(0) ? kl_term(m.x, softplus_sigma(r.x), a.x, b.x, conv) : 0.0f;
        s += w_in(1) ? kl_term(m.y, softplus_sigma(r.y), a.y, b.y, conv) : 0.0f;
        s += w_in(2) ? kl_term(m.z, softplus_sigma(r.z), a.z, b.z, conv) : 0.0f;
        s += w_in(3) ? kl_term(m.w, softplus_sigma(r.w), a.w, b.w, conv) : 0.0f;
        acc += (double)s;
    }
    for (uint64_t i = (n4 << 2) + tid; i < n_w; i += nth) {
        const float2 pr = TP ? make_float2(__ldg(q.w_mu + i), __ldg(q.w_sigma + i)) : make_float2(pm, ps);
        acc += kept(w_keep<MK>(q, i)) ? (double)kl_term(__ldg(w_mu + i), softplus_sigma(__ldg(w_rho + i)), pr.x, pr.y, conv)
                                      : 0.0;
    }
    for (uint64_t i = tid; i < n_b; i += nth) {
        const float2 pr = TP ? make_float2(__ldg(q.b_mu + i), __ldg(q.b_sigma + i)) : make_float2(pm, ps);
        acc += kept(b_keep<MK>(q, i)) ? (double)kl_term(__ldg(b_mu + i), softplus_sigma(__ldg(b_rho + i)), pr.x, pr.y, conv)
                                      : 0.0;
    }
    const double tot = block_sum(acc, red);
    if (threadIdx.x == 0) kl_publish(tot, blockIdx.x, gridDim.x, partials, counter, kl_out);
}

__global__ void __launch_bounds__(256)
kl_forward_kernel(const float* __restrict__ w_mu, const float* __restrict__ w_rho, uint64_t n_w,
                  const float* __restrict__ b_mu, const float* __restrict__ b_rho, uint64_t n_b,
                  float pm, float ps, int conv, double* partials, unsigned int* counter, float* kl_out) {
    kl_forward_body<false>(w_mu, w_rho, n_w, b_mu, b_rho, n_b, pm, ps, PriorPtrs{}, conv, partials, counter, kl_out);
}
__global__ void __launch_bounds__(256)
kl_forward_prior_kernel(const float* __restrict__ w_mu, const float* __restrict__ w_rho, uint64_t n_w,
                        const float* __restrict__ b_mu, const float* __restrict__ b_rho, uint64_t n_b,
                        const PriorPtrs q, int conv, double* partials, unsigned int* counter, float* kl_out) {
    kl_forward_body<true>(w_mu, w_rho, n_w, b_mu, b_rho, n_b, 0.0f, 1.0f, q, conv, partials, counter, kl_out);
}
// a masked layer (q.w_mask set); TP: against q's tensor prior, else the scalar (pm, ps)
template <bool TP>
__global__ void __launch_bounds__(256)
kl_forward_masked_kernel(const float* __restrict__ w_mu, const float* __restrict__ w_rho, uint64_t n_w,
                         const float* __restrict__ b_mu, const float* __restrict__ b_rho, uint64_t n_b,
                         float pm, float ps, const PriorPtrs q, int conv, double* partials, unsigned int* counter,
                         float* kl_out) {
    kl_forward_body<TP, true>(w_mu, w_rho, n_w, b_mu, b_rho, n_b, pm, ps, q, conv, partials, counter, kl_out);
}

// d kl / d mu = (mu - pm) / sigma^2 ; d kl / d sigma = 1/sigma - ps^2/sigma^3 - (mu-pm)^2/sigma^3 ;
// d sigma / d rho = sigmoid(rho)   (SURVEY.md Appendix A; reference convention).
// TP: element i's prior is (q_mu[i], q_sigma[i]) instead of (pm, ps).  MK: nothing is added for a pruned element
// (mask[i] == 0).
template <bool TP, bool MK = false>
__device__ __forceinline__ void kl_backward_body(const float* __restrict__ mu, const float* __restrict__ rho, uint64_t n,
                                                 float pm_, float ps_, const float* __restrict__ q_mu,
                                                 const float* __restrict__ q_sigma, int conv,
                                                 const float* __restrict__ grad_kl, float* __restrict__ g_mu,
                                                 float* __restrict__ g_rho, const uint8_t* __restrict__ mask = nullptr) {
    const float go = __ldg(grad_kl);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (MK && !kept(KeepAt{mask, i})) continue;
        const float pm = TP ? __ldg(q_mu + i) : pm_, ps = TP ? __ldg(q_sigma + i) : ps_;
        const float m = mu[i], r = rho[i];
        const float s = softplus_sigma(r), d = m - pm;
        const float sg = 1.0f / (1.0f + expf(-r));
        float dm, ds;
        if (conv == BBB_KL_REFERENCE) {
            const float is = 1.0f / s, is3 = is * is * is;
            dm = d * is * is;
            ds = is - ps * ps * is3 - d * d * is3;
        } else {
            dm = d / (ps * ps);
            ds = -1.0f / s + s / (ps * ps);
        }
        g_mu[i] += go * dm;
        g_rho[i] += go * ds * sg;
    }
}

__global__ void __launch_bounds__(256)
kl_backward_kernel(const float* __restrict__ mu, const float* __restrict__ rho, uint64_t n, float pm, float ps,
                   int conv, const float* __restrict__ grad_kl, float* __restrict__ g_mu, float* __restrict__ g_rho) {
    kl_backward_body<false>(mu, rho, n, pm, ps, nullptr, nullptr, conv, grad_kl, g_mu, g_rho);
}
__global__ void __launch_bounds__(256)
kl_backward_prior_kernel(const float* __restrict__ mu, const float* __restrict__ rho, uint64_t n,
                         const float* __restrict__ q_mu, const float* __restrict__ q_sigma, int conv,
                         const float* __restrict__ grad_kl, float* __restrict__ g_mu, float* __restrict__ g_rho) {
    kl_backward_body<true>(mu, rho, n, 0.0f, 1.0f, q_mu, q_sigma, conv, grad_kl, g_mu, g_rho);
}
// masked elements (mask non-NULL); TP: against (q_mu, q_sigma), else the scalar (pm, ps)
template <bool TP>
__global__ void __launch_bounds__(256)
kl_backward_masked_kernel(const float* __restrict__ mu, const float* __restrict__ rho, uint64_t n, float pm, float ps,
                          const float* __restrict__ q_mu, const float* __restrict__ q_sigma, const uint8_t* __restrict__ mask,
                          int conv, const float* __restrict__ grad_kl, float* __restrict__ g_mu, float* __restrict__ g_rho) {
    kl_backward_body<TP, true>(mu, rho, n, pm, ps, q_mu, q_sigma, conv, grad_kl, g_mu, g_rho, mask);
}

__global__ void __launch_bounds__(256)
philox_fill_kernel(float* __restrict__ out, uint64_t n, NoiseKey key, uint64_t offset) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = normal1(offset + i, key);
}

// Backward of the LRT noise term, gv = grad_y * eps / (2 * act_std) (layers/BBB_LRT/BBBConv.py:75-79), with eps drawn
// again where the forward drew it: Philox stream of row b's sample (fold_key), NHWC element index
// ((first_image + b) * OHW + pix) * N + c.  grad_y, act_std and gv are NCHW [B, N, OHW].  The two multiplies and the
// division are rounded one by one, as the element-wise ops of a tensor library do it.
// VEC4 (N % 4 == 0): a thread takes the four channels one Philox call draws, at one pixel; consecutive threads take
// consecutive pixels, so each of its four loads and stores is coalesced.  Otherwise one thread per element, in NCHW order.
template <bool VEC4>
__global__ void __launch_bounds__(256)
lrt_noise_grad_kernel(const float* __restrict__ gy, const float* __restrict__ act_std, float* __restrict__ gv,
                      int B, int N, int OHW, NoiseKey key, const unsigned long long* stream_base, McFold fold) {
    const NoiseKey k0 = effective_key(key, stream_base);
    const unsigned per = VEC4 ? N / 4 : N;
    const unsigned total = (unsigned)B * per * (unsigned)OHW;           // <= B * N * OHW < 2^31 (make_geom)
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const unsigned pix = t % (unsigned)OHW, r = t / (unsigned)OHW;
        const unsigned c = r % per;
        const int b = (int)(r / per);
        int bi;
        const NoiseKey k = fold_key(k0, fold, b, bi);
        const uint64_t pos = ((uint64_t)bi * OHW + pix) * N;                // NHWC index of channel 0 at this pixel
        if constexpr (VEC4) {
            const float4 z = normal4((pos >> 2) + c, k);                    // channels 4c .. 4c+3 (pos % 4 == 0)
            const float e[4] = {z.x, z.y, z.z, z.w};
            const unsigned o = ((unsigned)b * N + 4 * c) * (unsigned)OHW + pix;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned oj = o + j * (unsigned)OHW;
                gv[oj] = __fdiv_rn(__fmul_rn(__ldg(gy + oj), e[j]), __fmul_rn(2.0f, __ldg(act_std + oj)));
            }
        } else {
            const float e = normal1(pos + c, k);
            gv[t] = __fdiv_rn(__fmul_rn(__ldg(gy + t), e), __fmul_rn(2.0f, __ldg(act_std + t)));
        }
    }
}

// The head of a captured Monte-Carlo step.  It lets its programmatic dependents start at once: the first GEMM kernel of
// a chain whose operand tiles are prepared ahead of the step stages its input images meanwhile, and every reader of the
// base waits (griddepcontrol.wait) for this kernel to complete.
__global__ void noise_advance_kernel(unsigned long long* base, unsigned long long inc) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    *base += inc;
}

// main_bayesian.py:46-53 + utils.py:14-22 (+ uncertainty_estimation.py:70-96 moments).
// One CTA per image; warps compute log-sum-exp per MC sample, then one thread per
// class folds the S samples with an online logmeanexp.
__global__ void __launch_bounds__(128)
mc_combine_kernel(const float* __restrict__ logits, int S, int B, int C, float* __restrict__ log_out,
                  float* __restrict__ moments) {
    extern __shared__ float lse[];            // [S]
    const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int s = wid; s < S; s += nw) {
        const float* row = logits + ((size_t)s * B + b) * C;
        float mx = -INFINITY;
        for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float se = 0.0f;
        for (int c = lane; c < C; c += 32) se += expf(row[c] - mx);
        se = warp_sum(se);
        if (lane == 0) lse[s] = mx + logf(se);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float mx = -INFINITY, acc = 0.0f, sp = 0.0f, sp2 = 0.0f, sl = 0.0f;
        for (int s = 0; s < S; ++s) {
            const float l = logits[((size_t)s * B + b) * C + c];
            const float v = l - lse[s];          // log_softmax
            if (v > mx) { acc = acc * expf(mx - v) + 1.0f; mx = v; }
            else if (v > -INFINITY) acc += expf(v - mx);   // v == -inf: a probability of 0 adds nothing (not exp(NaN))
            const float pr = expf(v);
            sp += pr; sp2 += pr * pr; sl += l;
        }
        log_out[(size_t)b * C + c] = mx + logf(acc / (float)S);
        if (moments) {
            const size_t bc = (size_t)B * C, o = (size_t)b * C + c;
            moments[o] = sp; moments[bc + o] = sp2; moments[2 * bc + o] = sl;
        }
    }
}

}  // namespace bbb
