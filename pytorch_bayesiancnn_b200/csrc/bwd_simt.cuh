// Backward of the Bayesian layer forward (SURVEY.md Appendix A), IEEE fp32 on CUDA cores.
//
//   BBB : W = mu + eps*sigma, y = x (*) W + b
//         G_W = wgrad(x, gy);  d mu = G_W;  d rho = G_W * eps * sigmoid(rho);  dx = dgrad(gy, W)
//   LRT : y = m + sqrt(v)*eps, m = x (*) mu + b_mu, v = 1e-16 + x^2 (*) sigma^2 + sigma_b^2
//         g_m = gy;  g_v = gy * eps / (2 sqrt(v));
//         d mu = wgrad(x, g_m);  d rho = 2 sigma sigmoid(rho) * wgrad(x^2, g_v);
//         dx = dgrad(g_m, mu) + 2 x * dgrad(g_v, sigma^2)
// eps is regenerated from the Philox stream of the forward (or re-read from the external eps
// tensors): nothing weight- or activation-sized is stored between forward and backward except
// the LRT sqrt(v) (act_std).
//
// Two kernels: wgrad (N x K tile, split over M with atomic accumulation, also reduces the bias
// gradients) and dgrad (implicit GEMM over input pixels).  Replaces the autograd graph of
// layers/BBB/BBBConv.py:61-77, BBB/BBBLinear.py:54-70, BBB_LRT/BBBConv.py:62-81, BBB_LRT/BBBLinear.py:56-73.
#pragma once
#include "common.cuh"

namespace bbb {

struct BwdArgs {
    Geom g;
    const float* x; const float* gy; const float* w_mu; const float* w_rho; const float* b_mu; const float* b_rho;
    const float* act_std; const float* eps_a; const float* eps_b;
    NoiseKey key; const unsigned long long* stream_base;
    float* gx; float* g_w_mu; float* g_w_rho; float* g_b_mu; float* g_b_rho;
    int sample, has_bias, variant;
    int m_chunk;        // rows of M per wgrad split
    int first_image;    // as in the forward (FwdArgs): LRT noise of image b is drawn at image first_image + b
    PriorPtrs prior;    // only the mask (w_mask, b_mask) is read, by the MK = true instantiations
};

__device__ __forceinline__ float sigmoidf_(float r) { return 1.0f / (1.0f + expf(-r)); }

// g_v = gy * eps / (2 sqrt(v)) at flat NCHW output index o = ((b*N + n)*OHW + pix)
__device__ __forceinline__ float lrt_gv(const BwdArgs& p, const NoiseKey& k, float gy, size_t o, int b, int n, int pix) {
    const float e = p.eps_a ? __ldg(p.eps_a + o) : normal1(((uint64_t)(b + p.first_image) * p.g.OHW + pix) * p.g.N + n, k);
    return gy * e / (2.0f * __ldg(p.act_std + o));
}

// --------------------------------------------------------------------- wgrad
// grid = (k tiles, n tiles, M splits); 256 threads; tile 64(n) x 64(k), reduction chunk 16 rows of M.
// MK: nothing is added to the gradients of a pruned element (p.prior.w_mask / b_mask), which stay exactly zero.
template <int VARIANT, bool MK = false>
__global__ void __launch_bounds__(256)
wgrad_simt_kernel(const BwdArgs p) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    constexpr int BK = 16, PAD = 4;
    __shared__ __align__(16) float Gs[BK][64 + PAD];                  // gy      [m][n]
    __shared__ __align__(16) float Gv[LRT ? BK : 1][64 + PAD];        // g_v     [m][n]
    __shared__ __align__(16) float As[BK][64 + PAD];                  // im2col  [m][k]
    const Geom& g = p.g;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    const bool stoch = p.sample != 0;
    const bool var_path = LRT && stoch;
    const int t = threadIdx.x;
    const int k0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
    const int m_begin = blockIdx.z * p.m_chunk, m_end = min(g.M, m_begin + p.m_chunk);
    const int lm = t & 15, lc = t >> 4;          // load mapping: row of the chunk, column (+16 per slot)
    const int tx = t & 15, ty = t >> 4;          // compute mapping: k = tx*4.., n = ty*4..
    float acc[4][4], accv[LRT ? 4 : 1][LRT ? 4 : 1];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[i][j] = 0.0f; if (LRT) accv[i][j] = 0.0f; }
    float bsum = 0.0f, bsumv = 0.0f;             // bias gradients (threads 0..63 of the k-tile-0 CTAs)

    for (int mb = m_begin; mb < m_end; mb += BK) {
        const int m = mb + lm;
        const bool mv = m < m_end;
        int b = 0, pix = 0, ih0 = 0, iw0 = 0;
        if (mv) {
            b = m / g.OHW; pix = m - b * g.OHW;
            const int oh = pix / g.OW, ow = pix - oh * g.OW;
            ih0 = oh * g.SH - g.PH; iw0 = ow * g.SW - g.PW;
        }
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int c = lc + 16 * s;
            // gy (and g_v) tile
            const int n = n0 + c;
            float gyv = 0.0f, gvv = 0.0f;
            if (mv && n < g.N) {
                const size_t o = ((size_t)b * g.N + n) * g.OHW + pix;
                gyv = __ldg(p.gy + o);
                if (var_path) gvv = lrt_gv(p, nkey, gyv, o, b, n, pix);
            }
            Gs[lm][c] = gyv;
            if (LRT) Gv[lm][c] = gvv;
            // im2col tile
            const int k = k0 + c;
            float a = 0.0f;
            if (mv && k < g.K) {
                const int ci = k / g.KHW, rs = k - ci * g.KHW;
                const int r = rs / g.KW, sx = rs - r * g.KW;
                const int ih = ih0 + r * g.DH, iw = iw0 + sx * g.DW;
                if ((unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W)
                    a = __ldg(p.x + ((size_t)b * g.Cin + ci) * g.HW + ih * g.W + iw);
            }
            As[lm][c] = a;
        }
        __syncthreads();
#pragma unroll
        for (int mm = 0; mm < BK; ++mm) {
            float a[4], gg[4], gv[LRT ? 4 : 1];
#pragma unroll
            for (int j = 0; j < 4; ++j) a[j] = As[mm][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i) { gg[i] = Gs[mm][ty * 4 + i]; if (LRT) gv[i] = Gv[mm][ty * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    acc[i][j] = fmaf(gg[i], a[j], acc[i][j]);
                    if (LRT) accv[i][j] = fmaf(gv[i], a[j] * a[j], accv[i][j]);
                }
        }
        if (blockIdx.x == 0 && t < 64) {
#pragma unroll
            for (int mm = 0; mm < BK; ++mm) { bsum += Gs[mm][t]; if (LRT) bsumv += Gv[mm][t]; }
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= g.N) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tx * 4 + j;
            if (k >= g.K) continue;
            const size_t wi = (size_t)n * g.K + k;
            if (!kept(w_keep<MK>(p.prior, wi))) continue;
            atomicAdd(p.g_w_mu + wi, acc[i][j]);
            if (stoch) {
                const float rho = __ldg(p.w_rho + wi);
                const float sp = sigmoidf_(rho);
                if (LRT) {
                    atomicAdd(p.g_w_rho + wi, accv[i][j] * 2.0f * softplus_sigma(rho) * sp);
                } else {
                    const float e = p.eps_a ? __ldg(p.eps_a + wi) : normal1(wi, nkey);
                    atomicAdd(p.g_w_rho + wi, acc[i][j] * e * sp);
                }
            }
        }
    }
    if (p.has_bias && blockIdx.x == 0 && t < 64 && n0 + t < g.N && kept(b_keep<MK>(p.prior, n0 + t))) {
        const int n = n0 + t;
        atomicAdd(p.g_b_mu + n, bsum);
        if (stoch) {
            const float rho = __ldg(p.b_rho + n);
            const float sp = sigmoidf_(rho);
            if (LRT) atomicAdd(p.g_b_rho + n, bsumv * 2.0f * softplus_sigma(rho) * sp);
            else {
                const float e = p.eps_b ? __ldg(p.eps_b + n) : normal1((uint64_t)g.N * g.K + n, nkey);
                atomicAdd(p.g_b_rho + n, bsum * e * sp);
            }
        }
    }
}

// --------------------------------------------------------------------- dgrad
// Implicit GEMM: rows m' = (b, ih, iw) input pixels, columns c = input channels,
// reduction k' = (n, r, s).  grid = (m' tiles, c tiles); 256 threads; 64 x 64 x 16 tiles.
// MK: a pruned weight is a zero operand (p.prior.w_mask).
template <int VARIANT, bool MK = false>
__global__ void __launch_bounds__(256)
dgrad_simt_kernel(const BwdArgs p) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    constexpr int BK = 16, PAD = 4;
    __shared__ __align__(16) float As[BK][64 + PAD];                  // gy gathered [k'][m']
    __shared__ __align__(16) float Av[LRT ? BK : 1][64 + PAD];        // g_v gathered
    __shared__ __align__(16) float Bs[BK][64 + PAD];                  // W (BBB: sampled; LRT: mu)   [k'][c]
    __shared__ __align__(16) float Bv[LRT ? BK : 1][64 + PAD];        // LRT: sigma^2
    const Geom& g = p.g;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    const bool stoch = p.sample != 0;
    const bool var_path = LRT && stoch;
    const int t = threadIdx.x;
    const int m0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
    const int Mi = g.B * g.HW, Kd = g.N * g.KHW;
    const int lk = t >> 6, lc = t & 63;          // load mapping: 4 k' rows per pass, 64 columns
    const int tx = t & 15, ty = t >> 4;          // compute: m' = tx*4.., c = ty*4..
    // the input pixel this thread gathers for
    const int mrow = m0 + lc;
    const bool mv = mrow < Mi;
    int b = 0, ih = 0, iw = 0;
    if (mv) { b = mrow / g.HW; const int q = mrow - b * g.HW; ih = q / g.W; iw = q - ih * g.W; }
    float acc[4][4], accv[LRT ? 4 : 1][LRT ? 4 : 1];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[i][j] = 0.0f; if (LRT) accv[i][j] = 0.0f; }

    for (int kb = 0; kb < Kd; kb += BK) {
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int kl = lk + 4 * s, k = kb + kl;
            float a = 0.0f, av = 0.0f, w = 0.0f, wv = 0.0f;
            if (k < Kd) {
                const int n = k / g.KHW, rs = k - n * g.KHW;
                const int r = rs / g.KW, sx = rs - r * g.KW;
                if (mv) {
                    const int th = ih + g.PH - r * g.DH, tw = iw + g.PW - sx * g.DW;
                    if (th >= 0 && tw >= 0 && th % g.SH == 0 && tw % g.SW == 0) {
                        const int oh = th / g.SH, ow = tw / g.SW;
                        if (oh < g.OH && ow < g.OW) {
                            const int pix = oh * g.OW + ow;
                            const size_t o = ((size_t)b * g.N + n) * g.OHW + pix;
                            a = __ldg(p.gy + o);
                            if (var_path) av = lrt_gv(p, nkey, a, o, b, n, pix);
                        }
                    }
                }
                const int c = c0 + lc;
                if (c < g.Cin && kept(w_keep<MK>(p.prior, ((size_t)n * g.Cin + c) * g.KHW + rs))) {
                    const size_t wi = ((size_t)n * g.Cin + c) * g.KHW + rs;
                    const float mu = __ldg(p.w_mu + wi);
                    if (LRT) {
                        w = mu;
                        if (var_path) { const float sg = softplus_sigma(__ldg(p.w_rho + wi)); wv = sg * sg; }
                    } else if (stoch) {
                        const float e = p.eps_a ? __ldg(p.eps_a + wi) : normal1(wi, nkey);
                        w = mu + e * softplus_sigma(__ldg(p.w_rho + wi));
                    } else w = mu;
                }
            }
            As[kl][lc] = a; Bs[kl][lc] = w;
            if (LRT) { Av[kl][lc] = av; Bv[kl][lc] = wv; }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[4], w[4], av[LRT ? 4 : 1], wv[LRT ? 4 : 1];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[kk][tx * 4 + i]; if (LRT) av[i] = Av[kk][tx * 4 + i]; }
#pragma unroll
            for (int j = 0; j < 4; ++j) { w[j] = Bs[kk][ty * 4 + j]; if (LRT) wv[j] = Bv[kk][ty * 4 + j]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
                    if (LRT) accv[i][j] = fmaf(av[i], wv[j], accv[i][j]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tx * 4 + i;
        if (m >= Mi) continue;
        const int bb = m / g.HW, q = m - bb * g.HW;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = c0 + ty * 4 + j;
            if (c >= g.Cin) continue;
            const size_t xi = ((size_t)bb * g.Cin + c) * g.HW + q;
            float v = acc[i][j];
            if (var_path) v += 2.0f * __ldg(p.x + xi) * accv[i][j];
            p.gx[xi] = v;
        }
    }
}

inline cudaError_t launch_bwd_simt(BwdArgs a, cudaStream_t st, int n_sm, int* n_launch) {
    const Geom& g = a.g;
    *n_launch = 0;
    const bool lrt = a.variant == BBB_VARIANT_LRT;
    {   // wgrad: enough M splits to fill the machine, at least 64 rows each
        const int kt = (g.K + 63) / 64, nt = (g.N + 63) / 64;
        int splits = (2 * n_sm + kt * nt - 1) / (kt * nt);
        const int max_splits = (g.M + 63) / 64;
        if (splits > max_splits) splits = max_splits;
        if (splits < 1) splits = 1;
        a.m_chunk = ((g.M + splits - 1) / splits + 15) / 16 * 16;
        splits = (g.M + a.m_chunk - 1) / a.m_chunk;
        dim3 grid(kt, nt, splits);
        if (a.prior.w_mask) {
            if (lrt) wgrad_simt_kernel<BBB_VARIANT_LRT, true><<<grid, 256, 0, st>>>(a);
            else     wgrad_simt_kernel<BBB_VARIANT_BBB, true><<<grid, 256, 0, st>>>(a);
        } else {
            if (lrt) wgrad_simt_kernel<BBB_VARIANT_LRT><<<grid, 256, 0, st>>>(a);
            else     wgrad_simt_kernel<BBB_VARIANT_BBB><<<grid, 256, 0, st>>>(a);
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        *n_launch += 1;
    }
    if (a.gx) {
        dim3 grid((g.B * g.HW + 63) / 64, (g.Cin + 63) / 64);
        if (a.prior.w_mask) {
            if (lrt) dgrad_simt_kernel<BBB_VARIANT_LRT, true><<<grid, 256, 0, st>>>(a);
            else     dgrad_simt_kernel<BBB_VARIANT_BBB, true><<<grid, 256, 0, st>>>(a);
        } else {
            if (lrt) dgrad_simt_kernel<BBB_VARIANT_LRT><<<grid, 256, 0, st>>>(a);
            else     dgrad_simt_kernel<BBB_VARIANT_BBB><<<grid, 256, 0, st>>>(a);
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        *n_launch += 1;
    }
    return cudaSuccess;
}

}  // namespace bbb
