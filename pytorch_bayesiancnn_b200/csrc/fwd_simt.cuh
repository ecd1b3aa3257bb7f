// Fused Bayesian layer forward on CUDA cores (IEEE fp32): the exact-arithmetic
// path (BBB_MATH_FP32) and the path for shapes too small for a wgmma tile.
//
// One kernel per layer call does everything the reference spreads over ~15-40
// aten launches (SURVEY.md 2a): sigma = log1p(exp(rho)), eps (external or
// in-kernel Philox), W = mu + eps*sigma (BBB) or the mean/variance pair of
// contractions on x and x^2 (LRT), the implicit-GEMM conv / linear, bias, the
// reparameterised output, an optional fused activation, and the closed-form KL
// reduced to one scalar.  Replaces layers/BBB/BBBConv.py:61-83,
// layers/BBB/BBBLinear.py:54-76, layers/BBB_LRT/BBBConv.py:62-87,
// layers/BBB_LRT/BBBLinear.py:56-79 and metrics.py:27-29.
#pragma once
#include "common.cuh"

namespace bbb {

struct FwdArgs {
    Geom g;
    const float* x; const float* w_mu; const float* w_rho; const float* b_mu; const float* b_rho;
    float* y; float* kl_out; float* act_std;
    const float* eps_a; const float* eps_b;
    NoiseKey key; const unsigned long long* stream_base;
    double* kl_partials; unsigned int* kl_counter;
    float prior_mu, prior_sigma;
    int sample, kl_convention, has_bias, act;
    int first_image;    // global index of image 0: LRT noise of image b is drawn at image first_image + b (McFold)
    PriorPtrs prior;    // tensor prior (TP = true instantiations only) and mask (MK = true instantiations only)
};

__device__ __noinline__ float apply_act(float v, int act) {
    if (act == BBB_ACT_SOFTPLUS) return v > 20.0f ? v : log1pf(expf(v));   // nn.Softplus(beta=1, threshold=20)
    if (act == BBB_ACT_RELU) return fmaxf(v, 0.0f);
    return v;
}

// TP: the KL terms are taken against the tensor prior p.prior (bbb_prior) instead of (prior_mu, prior_sigma).
// MK: p.prior.w_mask / b_mask prune: a pruned element is a zero operand (mean and variance) and adds no KL term.
template <int VARIANT, int BM, int BN, int TM, int TN, bool TP = false, bool MK = false>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
fwd_simt_kernel(const FwdArgs p) {
    constexpr int BK = 16, NT = (BM / TM) * (BN / TN), PAD = 4;
    constexpr int A_PER = BM * BK / NT, B_PER = BN * BK / NT;
    constexpr bool LRT = (VARIANT == BBB_VARIANT_LRT);
    static_assert(NT % BM == 0 && NT % BK == 0 && A_PER >= 1 && B_PER >= 1, "tile/thread mismatch");

    __shared__ __align__(16) float As[BK][BM + PAD];
    __shared__ __align__(16) float Bs[BK][BN + PAD];                 // BBB: sampled W ; LRT: mu
    __shared__ __align__(16) float Bv[LRT ? BK : 1][BN + PAD];       // LRT: sigma^2
    __shared__ double red[32];

    const Geom& g = p.g;
    const int t = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const bool do_kl = (blockIdx.x == 0) && (p.kl_out != nullptr);
    const bool stoch = p.sample != 0;
    const bool need_var = LRT && stoch;
    const float* __restrict__ x = p.x;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);

    // ---- A (im2col of x) load mapping -------------------------------------
    // conv: consecutive threads walk m (output pixels: contiguous-ish in x);
    // linear-like: consecutive threads walk k (contiguous in x).
    const bool klin = g.linear_like != 0;
    const int a_m = klin ? (t / BK) : (t % BM);
    const int a_k = klin ? (t % BK) : (t / BM);
    constexpr int A_MSTEP = NT / BK;   // linear-like: m advances per slot
    constexpr int A_KSTEP = NT / BM;   // conv: k advances per slot
    int ih0 = 0, iw0 = 0; long xb = 0; bool mvalid = false;
    if (!klin) {
        const int m = m0 + a_m;
        mvalid = m < g.M;
        if (mvalid) {
            const int b = m / g.OHW, pix = m - b * g.OHW;
            const int oh = pix / g.OW, ow = pix - oh * g.OW;
            ih0 = oh * g.SH - g.PH; iw0 = ow * g.SW - g.PW;
            xb = (long)b * g.Cin * g.HW;
        }
    }
    // ---- B (weights) load mapping: consecutive threads walk k (contiguous) --
    const int b_k = t % BK, b_n = t / BK;
    constexpr int B_NSTEP = NT / BK;

    float ra[A_PER], rb[B_PER], rv[LRT ? B_PER : 1];
    double kl_acc = 0.0;

    auto fetch = [&](int kt) {
#pragma unroll
        for (int i = 0; i < A_PER; ++i) {
            float v = 0.0f;
            if (klin) {
                const int m = m0 + a_m + i * A_MSTEP, k = kt * BK + a_k;
                if (m < g.M && k < g.K) v = __ldg(x + (long)m * g.K + k);
            } else {
                const int k = kt * BK + a_k + i * A_KSTEP;
                if (mvalid && k < g.K) {
                    const int c = k / g.KHW, rs = k - c * g.KHW;
                    const int r = rs / g.KW, s = rs - r * g.KW;
                    const int ih = ih0 + r * g.DH, iw = iw0 + s * g.DW;
                    if ((unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W)
                        v = __ldg(x + xb + (long)c * g.HW + ih * g.W + iw);
                }
            }
            ra[i] = v;
        }
#pragma unroll
        for (int i = 0; i < B_PER; ++i) {
            const int n = n0 + b_n + i * B_NSTEP, k = kt * BK + b_k;
            float w = 0.0f, s2 = 0.0f;
            if (n < g.N && k < g.K && kept(w_keep<MK>(p.prior, (size_t)n * g.K + k))) {
                const size_t wi = (size_t)n * g.K + k;
                const float mu = __ldg(p.w_mu + wi);
                float sigma = 0.0f;
                if (stoch || do_kl) sigma = softplus_sigma(__ldg(p.w_rho + wi));
                if (LRT) {
                    w = mu; s2 = sigma * sigma;
                } else if (stoch) {
                    const float e = p.eps_a ? __ldg(p.eps_a + wi) : normal1(wi, nkey);
                    w = mu + e * sigma;                               // BBB/BBBConv.py:65
                } else {
                    w = mu;
                }
                if (do_kl) {
                    const float2 q = prior_of(w_prior<TP>(p, p.prior, wi));
                    kl_acc += (double)kl_term(mu, sigma, q.x, q.y, p.kl_convention);
                }
            }
            rb[i] = w;
            if (LRT) rv[i] = s2;
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int i = 0; i < A_PER; ++i) {
            if (klin) As[a_k][a_m + i * A_MSTEP] = ra[i];
            else      As[a_k + i * A_KSTEP][a_m] = ra[i];
        }
#pragma unroll
        for (int i = 0; i < B_PER; ++i) {
            Bs[b_k][b_n + i * B_NSTEP] = rb[i];
            if (LRT) Bv[b_k][b_n + i * B_NSTEP] = rv[i];
        }
    };

    const int tx = t % (BM / TM), ty = t / (BM / TM);
    float acc[TM][TN], accv[LRT ? TM : 1][LRT ? TN : 1];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) { acc[i][j] = 0.0f; if (LRT) accv[i][j] = 0.0f; }

    const int nk = (g.K + BK - 1) / BK;
    fetch(0);
    stash();
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        if (kt + 1 < nk) fetch(kt + 1);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[TM], b[TN], s2[LRT ? TN : 1];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = As[kk][tx * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) { b[j] = Bs[kk][ty * TN + j]; if (LRT) s2[j] = Bv[kk][ty * TN + j]; }
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                const float a2 = a[i] * a[i];
#pragma unroll
                for (int j = 0; j < TN; ++j) {
                    acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
                    if (LRT) accv[i][j] = fmaf(a2, s2[j], accv[i][j]);
                }
            }
        }
        __syncthreads();
        if (kt + 1 < nk) { stash(); __syncthreads(); }
    }

    // ---- bias (and its KL) --------------------------------------------------
    float bias_m[TN], bias_v[LRT ? TN : 1];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        const int n = n0 + ty * TN + j;
        float bm = 0.0f, bv = 0.0f;
        if (p.has_bias && n < g.N && kept(b_keep<MK>(p.prior, n))) {
            const float mu = __ldg(p.b_mu + n);
            if (stoch) {
                const float sigma = softplus_sigma(__ldg(p.b_rho + n));
                if (LRT) { bm = mu; bv = sigma * sigma; }
                else {
                    const float e = p.eps_b ? __ldg(p.eps_b + n) : normal1((uint64_t)g.N * g.K + n, nkey);
                    bm = mu + e * sigma;                              // BBB/BBBConv.py:70
                }
            } else {
                bm = mu;
            }
        }
        bias_m[j] = bm;
        if (LRT) bias_v[j] = bv;
    }
    if (do_kl) {
        if (p.has_bias && t < BN && n0 + t < g.N && kept(b_keep<MK>(p.prior, n0 + t))) {
            const float mu = __ldg(p.b_mu + n0 + t), sigma = softplus_sigma(__ldg(p.b_rho + n0 + t));
            const float2 q = prior_of(b_prior<TP>(p, p.prior, (size_t)(n0 + t)));
            kl_acc += (double)kl_term(mu, sigma, q.x, q.y, p.kl_convention);
        }
        const double tot = block_sum(kl_acc, red);
        if (t == 0) kl_publish(tot, blockIdx.y, gridDim.y, p.kl_partials, p.kl_counter, p.kl_out);
    }

    // ---- epilogue: reparameterise, activate, store NCHW ----------------------
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + tx * TM + i;
        if (m >= g.M) continue;
        const int b = m / g.OHW, pix = m - b * g.OHW;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + ty * TN + j;
            if (n >= g.N) continue;
            const size_t o = ((size_t)b * g.N + n) * g.OHW + pix;
            float v = acc[i][j] + bias_m[j];
            if (need_var) {
                const float var = 1e-16f + (accv[i][j] + bias_v[j]);   // BBB_LRT/BBBConv.py:73-74
                const float sd = sqrtf(var);
                // Philox element index of the activation noise: NHWC-flat ((b*OHW + pix)*N + n), b counted from first_image
                const float e = p.eps_a ? __ldg(p.eps_a + o)
                                        : normal1(((uint64_t)(b + p.first_image) * g.OHW + pix) * g.N + n, nkey);
                v = v + sd * e;                                       // BBB_LRT/BBBConv.py:79
                if (p.act_std) p.act_std[o] = sd;
            }
            p.y[o] = apply_act(v, p.act);
        }
    }
}

template <int VARIANT, int BM, int BN, int TM, int TN, bool TP, bool MK>
inline cudaError_t launch_fwd_simt_cfg(const FwdArgs& a, cudaStream_t st) {
    dim3 grid((a.g.M + BM - 1) / BM, (a.g.N + BN - 1) / BN);
    fwd_simt_kernel<VARIANT, BM, BN, TM, TN, TP, MK><<<grid, (BM / TM) * (BN / TN), 0, st>>>(a);
    return cudaGetLastError();
}

inline int simt_n_tile(int N) { return N <= 16 ? 16 : (N <= 32 ? 32 : 64); }
inline int simt_kl_slots(const Geom& g) { const int bn = simt_n_tile(g.N); return (g.N + bn - 1) / bn; }

template <int VARIANT, bool TP, bool MK>
inline cudaError_t launch_fwd_simt_tp(const FwdArgs& a, cudaStream_t st) {
    const int bn = simt_n_tile(a.g.N);
    if (bn == 16) return launch_fwd_simt_cfg<VARIANT, 128, 16, 4, 2, TP, MK>(a, st);
    if (bn == 32) return launch_fwd_simt_cfg<VARIANT, 128, 32, 4, 4, TP, MK>(a, st);
    return launch_fwd_simt_cfg<VARIANT, 64, 64, 4, 4, TP, MK>(a, st);
}
// a tensor prior (a.prior.w_mu, set only when the call computes a KL) takes the TP instantiations, a mask
// (a.prior.w_mask) the MK ones
template <int VARIANT>
inline cudaError_t launch_fwd_simt(const FwdArgs& a, cudaStream_t st) {
    return prior_dispatch(a.prior, [&](auto tp, auto mk) {
        return launch_fwd_simt_tp<VARIANT, decltype(tp)::value, decltype(mk)::value>(a, st);
    });
}

}  // namespace bbb
