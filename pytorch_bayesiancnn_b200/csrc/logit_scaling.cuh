// Vector and matrix scaling of the Monte-Carlo predictive (Guo et al. 2017), applied per sample before the softmax and
// the average over samples, as the temperature is (temperature.cuh):  p_bar = mean_s softmax(a . z_s + b) or
// mean_s softmax(W z_s + b) (include/bbb_b200.h, bbb_mc_logit_scale / bbb_scaling_nll_grad).  Vector scaling:
//
//  (A) mc_logit_scale_kernel   -- z <- a . z + b in place on a step's [S_local, rows, C] logits, a and b read from device
//      memory at run time; __fmul_rn then __fadd_rn (never contracted to an FMA): the bits of torch's fp32 z * a + b.
//  (G) scaling_nll_grad_kernel -- one full-batch pass over a logit bank (temperature.cuh's layout): the objective
//          J(a, b) = -(1/n) sum_i log( (1/S) sum_s softmax(a . z_is + b)[y_i] ) + mu sum_c b_c^2 / C,
//      its gradient and one Adam step of (a, b), in one launch.
//      One warp per image (TN_IMAGES images per warp, a CTA per fixed block of SC_CTA_IMAGES images, a function of the
//      image index alone, as temperature_nll_kernel):
//        pass 1, one lane per sample row s (as temperature_nll_kernel; the lanes' loads are C floats apart): m_s =
//        max_c z'_sc, l_s = log2 sum_c exp2((z'_sc - m_s) log2 e) summed over c in order, lp_s = log p_s[y];
//        then, in double over s: L_i = logmeanexp_s lp_s and the weights w_s = p_s[y] / sum_s' p_s'[y];
//        pass 2, lanes over the classes (coalesced), s in order: g_sc = w_s (1[c = y] - p_sc),
//        dL_i/da_c += g_sc z_sc, dL_i/db_c += g_sc.
//      Per-image sums are double, in each warp's own shared accumulators (a lane owns its classes), then over the warps
//      and over the CTAs in index order by the last CTA to arrive: the same bits on every run and for any bank capacity.
//      That CTA finishes the objective and gradient, tracks the best iterate and takes the Adam step.
#pragma once
#include "common.cuh"
#include "fwd_tc.cuh"       // pdl_wait / pdl_trigger
#include "temperature.cuh"  // ex2_ftz, TN_IMAGES

namespace bbb {

// ---- (A) apply -------------------------------------------------------------------------------------------------
constexpr int LS_THREADS = 256, LS_MAX_CTAS = 1024;

// Element j of the flat [rows][C] view is class j % C; a thread steps its class by the grid stride mod C, so the loop
// divides nothing.  Launched with programmatic serialization behind the kernel that writes z.
__global__ void __launch_bounds__(LS_THREADS)
mc_logit_scale_kernel(float* z, long long n, int C, const float* params /* a [C], b [C] */) {
    pdl_wait();
    pdl_trigger();
    const long long tid = (long long)blockIdx.x * LS_THREADS + threadIdx.x, stride = (long long)gridDim.x * LS_THREADS;
    const int step = (int)(stride % C);
    int c = (int)(tid % C);
    for (long long j = tid; j < n; j += stride) {
        z[j] = __fadd_rn(__fmul_rn(z[j], __ldg(params + c)), __ldg(params + C + c));
        c += step;
        if (c >= C) c -= C;
    }
}

// ---- (G) objective, gradient and Adam step ---------------------------------------------------------------------
constexpr int SC_THREADS = 256, SC_WARPS = SC_THREADS / 32;
constexpr int SC_CTA_IMAGES = SC_WARPS * TN_IMAGES;
constexpr int SC_MAX_S = 256;
static_assert(SC_CTA_IMAGES == BBB_SCALING_CTA_IMAGES && SC_MAX_S == BBB_LOGIT_BANK_MAX_SAMPLES,
              "vector scaling fit: header and kernel disagree");
constexpr double SC_BETA1 = 0.9, SC_BETA2 = 0.999, SC_EPS = 1e-8;
__device__ __forceinline__ double sc_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

// butterfly maxima: every lane ends with the same value
__device__ __forceinline__ float sc_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double sc_warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct ScalingNllArgs {
    const float* logits;                        // [n][S][C]
    const long long* labels;                    // [n]
    const long long* cursor;                    // nullable: images = min(cursor[0], n); cursor[1] > 0 poisons
    int n, S, C, first, last, update, matrix;
    float* theta;                               // [P]: the iterate this pass evaluates (fp32, as applied); P = 2C
                                                // (vector: a, b) or C^2 + C (matrix: W row by row, b)
    double* state;                              // [3][P]: Adam's double iterate, first and second moments
    float* best;                                // [P]: the best iterate so far
    double* fit;                                // [3]: objective at the start, the best objective, this pass's objective
    double* result;                             // [1 + P], nullable: this pass's objective and gradient
    float* out;                                 // [P]: the last pass writes the best iterate here, when there is a fit
    double l2_offdiag, l2_bias, lr, bias1, bias2;   // lambda, mu; the Adam step's rate and bias corrections 1 - beta^t
    double* partials;                           // [gridDim.x][1 + P]
    unsigned int* arrive;                       // zero between launches (the last CTA resets it)
};

// The last CTA of a pass: the sums over the CTAs' partials in index order (into tot [1 + P] of shared memory), the
// objective with its penalties, the gradient, the best iterate, the Adam step and, on the last pass, the result.
// Parameters: vector [a (C) | b (C)], matrix [W (C x C, row j = output j) | b (C)].
__device__ void sc_finish(const ScalingNllArgs& a, double* tot, int nthreads, long long n_img, bool poisoned) {
    __shared__ double obj_sh;
    __shared__ int improved_sh, finite_sh;
    const int C = a.C, nw = a.matrix ? C * C : C, P = nw + C;
    for (int j = threadIdx.x; j <= P; j += nthreads) {
        double t = 0.0;
#pragma unroll 16
        for (int b = 0; b < (int)gridDim.x; ++b) t += __ldcg(a.partials + (size_t)b * (P + 1) + j);
        tot[j] = t;
    }
    __syncthreads();
    const double inv_n = 1.0 / (double)n_img, off = a.matrix && C > 1 ? (double)C * (double)(C - 1) : 1.0;
    if (threadIdx.x == 0) {
        double reg_b = 0.0, reg_w = 0.0;
        for (int c = 0; c < C; ++c) reg_b += (double)a.theta[nw + c] * (double)a.theta[nw + c];
        if (a.matrix)
            for (int j = 0; j < nw; ++j)
                if (j / C != j % C) reg_w += (double)a.theta[j] * (double)a.theta[j];
        const double obj = (poisoned || n_img < 1) ? sc_nan()
                           : -tot[0] * inv_n + a.l2_offdiag * reg_w / off + a.l2_bias * reg_b / (double)C;
        const bool improved = a.first || obj < a.fit[1];
        if (a.first) a.fit[0] = obj;
        if (improved) a.fit[1] = obj;
        a.fit[2] = obj;
        if (a.result) a.result[0] = obj;
        obj_sh = obj;
        improved_sh = improved;
        finite_sh = isfinite(a.fit[0]) && isfinite(a.fit[1]);
        *a.arrive = 0u;
    }
    __syncthreads();
    const bool finite = isfinite(obj_sh);
    for (int j = threadIdx.x; j < P; j += nthreads) {
        const double th = (double)a.theta[j];
        const double pen = j >= nw ? 2.0 * a.l2_bias * th / (double)C
                         : (a.matrix && j / C != j % C) ? 2.0 * a.l2_offdiag * th / off : 0.0;
        const double g = -tot[1 + j] * inv_n + pen;
        if (a.result) a.result[1 + j] = g;
        if (improved_sh) a.best[j] = a.theta[j];
        if (a.update && finite) {
            double* x = a.state;
            double* m1 = a.state + P;
            double* m2 = a.state + 2 * P;
            const double mj = SC_BETA1 * m1[j] + (1.0 - SC_BETA1) * g;
            const double vj = SC_BETA2 * m2[j] + (1.0 - SC_BETA2) * g * g;
            m1[j] = mj;
            m2[j] = vj;
            x[j] -= a.lr * (mj / a.bias1) / (sqrt(vj / a.bias2) + SC_EPS);
            a.theta[j] = (float)x[j];
        }
        if (a.last && finite_sh) a.out[j] = a.best[j];
    }
}

inline size_t sc_smem_bytes(int C) { return (size_t)2 * C * sizeof(float) + (size_t)SC_WARPS * 2 * C * sizeof(double); }

__global__ void __launch_bounds__(SC_THREADS)
scaling_nll_grad_kernel(const ScalingNllArgs a) {
    extern __shared__ double dyn_sh[];
    double* acc_sh = dyn_sh;                                        // [SC_WARPS][2C]: per-warp sums of dL_i/d(a, b)
    float* th_sh = reinterpret_cast<float*>(dyn_sh + (size_t)SC_WARPS * 2 * a.C);   // [2C]: a, b
    __shared__ float m_sh[SC_WARPS][SC_MAX_S], l_sh[SC_WARPS][SC_MAX_S], w_sh[SC_WARPS][SC_MAX_S];
    __shared__ double ll_sh[SC_WARPS];
    __shared__ int last_sh;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, C = a.C, P = 2 * C;
    for (int j = threadIdx.x; j < P; j += SC_THREADS) th_sh[j] = a.theta[j];
    for (int j = threadIdx.x; j < SC_WARPS * P; j += SC_THREADS) acc_sh[j] = 0.0;
    long long n_img = a.n;
    bool poisoned = false;
    if (a.cursor) {
        n_img = min(a.cursor[0], (long long)a.n);
        poisoned = a.cursor[1] != 0;
    }
    __syncthreads();
    const float L2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
    const double ln_s = log((double)a.S);
    double* acc = acc_sh + (size_t)warp * P;
    double ll_acc = 0.0;                                            // this warp's sum of L_i (lane 0's is used)
    for (int j = 0; j < TN_IMAGES; ++j) {
        const long long i = (long long)blockIdx.x * SC_CTA_IMAGES + warp * TN_IMAGES + j;
        if (i >= n_img) break;
        __syncwarp();                                               // the last image's pass 2 has read the row stats
        const long long y = a.labels[i];
        const bool ok = y >= 0 && y < C;
        const float* img = a.logits + (size_t)i * a.S * C;
        // pass 1: one lane per sample row (s = lane, lane + 32, ..): the max, log2 of the normaliser and log p_s[y]
        for (int s = lane; s < a.S; s += 32) {
            const float* row = img + (size_t)s * C;
            float m = -INFINITY;
#pragma unroll 8
            for (int c = 0; c < C; ++c) m = fmaxf(m, __fadd_rn(__fmul_rn(__ldg(row + c), th_sh[c]), th_sh[C + c]));
            float e = 0.0f;
#pragma unroll 8
            for (int c = 0; c < C; ++c)
                e += ex2_ftz((__fadd_rn(__fmul_rn(__ldg(row + c), th_sh[c]), th_sh[C + c]) - m) * L2E);
            const float l2 = log2f(e);
            const float ty = ok ? __fadd_rn(__fmul_rn(__ldg(row + y), th_sh[y]), th_sh[C + y]) : m;
            m_sh[warp][s] = m;
            l_sh[warp][s] = l2;
            w_sh[warp][s] = (ty - m) - l2 * LN2;                    // lp_s, replaced by w_s below
        }
        __syncwarp();
        // the logmeanexp over s and the weights, in double
        double M = -INFINITY;
        for (int s = lane; s < a.S; s += 32) M = fmax(M, (double)w_sh[warp][s]);
        M = sc_warp_max(M);
        double Q = 0.0;
        for (int s = lane; s < a.S; s += 32) Q += exp((double)w_sh[warp][s] - M);
        Q = warp_sum(Q);
        __syncwarp();
        for (int s = lane; s < a.S; s += 32) w_sh[warp][s] = (float)(exp((double)w_sh[warp][s] - M) / Q);
        __syncwarp();
        ll_acc += ok ? M + log(Q) - ln_s : sc_nan();
        if (!ok) continue;
        // pass 2: per class, the gradient of L_i
        for (int c = lane; c < C; c += 32) {
            const float ac = th_sh[c], bc = th_sh[C + c];
            double da = 0.0, db = 0.0;
#pragma unroll 8
            for (int s = 0; s < a.S; ++s) {                         // (unrolled: the loads of 8 rows in flight)
                const float z = __ldg(img + (size_t)s * C + c);
                const float t = __fadd_rn(__fmul_rn(z, ac), bc);
                const float p = ex2_ftz((t - m_sh[warp][s]) * L2E - l_sh[warp][s]);
                const double g = (double)w_sh[warp][s] * ((c == y ? 1.0 : 0.0) - (double)p);
                da += g * (double)z;
                db += g;
            }
            acc[c] += da;
            acc[C + c] += db;
        }
    }
    if (lane == 0) ll_sh[warp] = ll_acc;
    __syncthreads();
    double* part = a.partials + (size_t)blockIdx.x * (P + 1);
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < SC_WARPS; ++w) t += ll_sh[w];
        part[0] = t;
    }
    for (int j = threadIdx.x; j < P; j += SC_THREADS) {
        double t = 0.0;
        for (int w = 0; w < SC_WARPS; ++w) t += acc_sh[(size_t)w * P + j];
        part[1 + j] = t;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last_sh = atomicAdd(a.arrive, 1u) == gridDim.x - 1u;
    __syncthreads();
    if (!last_sh) return;
    __threadfence();
    sc_finish(a, acc_sh, SC_THREADS, n_img, poisoned);           // (the per-warp accumulators hold the 1 + 2C sums)
}

// ---- (M) matrix scaling: z' = W z + b, C <= MX_MAX_C ------------------------------------------------------------
constexpr int MX_MAX_C = 128;
static_assert(MX_MAX_C == BBB_SCALING_MATRIX_MAX_CLASSES, "matrix scaling: header and kernel disagree");
constexpr int MA_THREADS = 128, MA_ROWS = 8, MA_MAX_CTAS = 1024;

// The apply: a CTA stages W^T once (shared, [k][j]) and then MA_ROWS rows of z at a time; thread j forms output j of
// each row as acc = fmaf(W[j][k], z[k], acc) for k = 0, 1, .., C-1 from acc = 0, then acc + b[j] (__fadd_rn), the
// MA_ROWS rows' chains side by side, and the rows are written back in place once all of them are staged.  Launched behind the logits' producer with PDL.
__global__ void __launch_bounds__(MA_THREADS)
mc_logit_scale_matrix_kernel(float* z, long long rows, int C, const float* params /* W [C][C], b [C] */) {
    extern __shared__ float ma_sh[];
    float* wt = ma_sh;                                              // [C][C]: wt[k * C + j] = W[j][k]
    float* zr = ma_sh + C * C;                                      // [MA_ROWS][C]
    pdl_wait();
    pdl_trigger();
    for (int e = threadIdx.x; e < C * C; e += MA_THREADS) {
        const int j = e / C, k = e - j * C;
        wt[k * C + j] = __ldg(params + e);
    }
    const int j = threadIdx.x;
    const float bj = j < C ? __ldg(params + C * C + j) : 0.0f;
    for (long long r0 = (long long)blockIdx.x * MA_ROWS; r0 < rows; r0 += (long long)gridDim.x * MA_ROWS) {
        const int nr = (int)min((long long)MA_ROWS, rows - r0);
        __syncthreads();                                            // (W^T staged; the last group's rows consumed)
        for (int e = threadIdx.x; e < nr * C; e += MA_THREADS) zr[e] = z[r0 * C + e];
        __syncthreads();
        if (j < C) {
            float acc[MA_ROWS];
#pragma unroll
            for (int r = 0; r < MA_ROWS; ++r) acc[r] = 0.0f;
            for (int k = 0; k < C; ++k) {
                const float w = wt[k * C + j];
#pragma unroll
                for (int r = 0; r < MA_ROWS; ++r) acc[r] = fmaf(w, zr[(r < nr ? r : 0) * C + k], acc[r]);
            }
#pragma unroll
            for (int r = 0; r < MA_ROWS; ++r)
                if (r < nr) z[(r0 + r) * C + j] = __fadd_rn(acc[r], bj);
        }
    }
}

// The fit pass of matrix scaling, on tf32 wgmma with fp32 accumulation (one warpgroup per CTA):
//   forward   Z' = Z W^T + b over 64-row tiles of the bank's rows (A = the Z tile [64][Kc], B = W [128][Kc], K-major,
//             both tf32-rounded; the accumulator stays in registers and b is added in fp32);
//   epilogue  per row, across the quad of lanes that holds it: the max, log2 of the normaliser, log p[y]; after all
//             of a CTA's rows the logmeanexp over each image's samples and the weights w_s in double (as the vector
//             pass); a second sweep recomputes Z' and writes G = w_s (1[c = y] - p) as tf32 into G^T [128][64];
//   gradient  dW += G^T Z per tile (A = G^T, B = Z^T [128][64], K = the 64 rows), fp32 accumulators in registers
//             across the CTA's tiles; db = sum over rows of the tf32 G, in double in row order.
// A CTA takes mx_images(S) consecutive images (a function of S and the image index alone); its partials are summed over
// the CTAs in index order by the last one to arrive (sc_finish).  Operand layout: fwd_tc.cuh's K-major SWIZZLE_NONE
// core matrices, 16-byte chunk q of row r at q * rows * 16 + r * 16.
constexpr int MX_THREADS = 128, MX_TM = 64, MX_N = 128, MX_ROWS = 2048;
// shared memory, sized by Kc = C rounded up to 8 (so that small C runs several CTAs per SM):
// [W: 128 x Kc][Z tile: 64 x Kc][Z^T: 128 x 64][G^T: 128 x 64][m, l, w: 3 x MX_ROWS fp32]
constexpr size_t MX_T_BYTES = (size_t)MX_N * MX_TM * 4;
__host__ __device__ inline size_t mx_w_bytes(int Kc) { return (size_t)MX_N * Kc * 4; }
__host__ __device__ inline size_t mx_z_bytes(int Kc) { return (size_t)MX_TM * Kc * 4; }
__host__ __device__ inline size_t mx_stat_off(int Kc) { return mx_w_bytes(Kc) + mx_z_bytes(Kc) + 2 * MX_T_BYTES; }
inline size_t mx_smem_bytes(int C) { return 1024 + mx_stat_off((C + 7) & ~7) + (size_t)3 * MX_ROWS * 4; }
__host__ __device__ inline int mx_images(int S) { return MX_ROWS / S > 1 ? MX_ROWS / S : 1; }
__device__ __forceinline__ uint32_t mx_off(int rows, int r, int k) {
    return (uint32_t)(k >> 2) * (uint32_t)rows * 16u + (uint32_t)r * 16u + (uint32_t)(k & 3) * 4u;
}

__global__ void __launch_bounds__(MX_THREADS)
scaling_nll_grad_matrix_kernel(const ScalingNllArgs a) {
    extern __shared__ uint8_t mx_raw[];
    const uint32_t raw = smem_u32(mx_raw), base = (raw + 1023u) & ~1023u;
    uint8_t* gb = mx_raw + (base - raw);
    const int Kc = (a.C + 7) & ~7;
    const uint32_t w_op = base, z_op = base + (uint32_t)mx_w_bytes(Kc), zt_op = z_op + (uint32_t)mx_z_bytes(Kc),
                   gt_op = zt_op + (uint32_t)MX_T_BYTES;
    uint8_t *w_g = gb, *z_g = gb + mx_w_bytes(Kc), *zt_g = z_g + mx_z_bytes(Kc), *gt_g = zt_g + MX_T_BYTES;
    float* m_sh = reinterpret_cast<float*>(gb + mx_stat_off(Kc));
    float* l_sh = m_sh + MX_ROWS;
    float* w_sh = l_sh + MX_ROWS;
    __shared__ float b_sh[MX_N];
    __shared__ double ll_sh[MX_THREADS / 32];
    __shared__ int last_sh;
    const int t = threadIdx.x, warp = t >> 5, l = t & 31, C = a.C, S = a.S, nw = C * C;
    for (int e = t; e < MX_N * Kc; e += MX_THREADS) {               // W [128][Kc], zero-padded
        const int j = e / Kc, k = e - j * Kc;
        const float v = (j < C && k < C) ? a.theta[j * C + k] : 0.0f;
        *reinterpret_cast<uint32_t*>(w_g + mx_off(MX_N, j, k)) = to_tf32(v);
    }
    for (int e = t; e < (int)(MX_T_BYTES / 4); e += MX_THREADS) reinterpret_cast<float*>(zt_g)[e] = 0.0f;
    b_sh[t] = t < C ? a.theta[nw + t] : 0.0f;
    long long n_img = a.n;
    bool poisoned = false;
    if (a.cursor) {
        n_img = min(a.cursor[0], (long long)a.n);
        poisoned = a.cursor[1] != 0;
    }
    const int IMG = mx_images(S);
    const long long img0 = (long long)blockIdx.x * IMG;
    const int nimg = (int)max(0ll, min((long long)IMG, n_img - img0));
    const int R = nimg * S, tiles = (R + MX_TM - 1) / MX_TM;
    const float* zb = a.logits + (size_t)img0 * S * C;
    const float L2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

    auto load_tile = [&](int tt, bool transposed) {
        for (int e = t; e < MX_TM * Kc; e += MX_THREADS) {
            const int rr = e / Kc, k = e - rr * Kc, r = tt * MX_TM + rr;
            const uint32_t u = to_tf32((r < R && k < C) ? __ldg(zb + (size_t)r * C + k) : 0.0f);
            *reinterpret_cast<uint32_t*>(z_g + mx_off(MX_TM, rr, k)) = u;
            if (transposed) *reinterpret_cast<uint32_t*>(zt_g + mx_off(MX_N, k, rr)) = u;
        }
        fence_proxy_async();                                        // generic-proxy writes -> the tensor core
        __syncthreads();
    };
    auto forward = [&](float (&d0)[32], float (&d1)[32]) {
        wgmma_fence();
        for (int ks = 0; ks < Kc / 8; ++ks) {
            const uint64_t da = make_smem_desc(z_op + (uint32_t)ks * 2u * MX_TM * 16u, MX_TM * 16, 128);
            const uint64_t db0 = make_smem_desc(w_op + (uint32_t)ks * 2u * MX_N * 16u, MX_N * 16, 128);
            const uint64_t db1 = make_smem_desc(w_op + (uint32_t)ks * 2u * MX_N * 16u + 64u * 16u, MX_N * 16, 128);
            wgmma_m64n64k8_tf32(d0, da, db0, ks > 0 ? 1u : 0u);
            wgmma_m64n64k8_tf32(d1, da, db1, ks > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
    };
    // the label of tile row rl's image (-1 past the CTA's rows)
    auto label_of = [&](int r) -> long long { return r < R ? a.labels[img0 + r / S] : -1ll; };

    // sweep 1: the row statistics
    __syncthreads();
    for (int tt = 0; tt < tiles; ++tt) {
        __syncthreads();                                            // the last tile's operands are consumed
        load_tile(tt, false);
        float d0[32], d1[32];
        forward(d0, d1);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int r = tt * MX_TM + 16 * warp + (l >> 2) + 8 * hr;
            const long long y = label_of(r);
            float m = -INFINITY, ty = 0.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 64 * h + 8 * jj + 2 * (l & 3) + e;
                        const float v = (h ? d1 : d0)[4 * jj + 2 * hr + e] + b_sh[c];
                        if (c < C) m = fmaxf(m, v);
                        if (c == y) ty = v;
                    }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            float sum = 0.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 64 * h + 8 * jj + 2 * (l & 3) + e;
                        const float v = (h ? d1 : d0)[4 * jj + 2 * hr + e] + b_sh[c];
                        if (c < C) sum += ex2_ftz((v - m) * L2E);
                    }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            ty += __shfl_xor_sync(0xffffffffu, ty, 1);
            ty += __shfl_xor_sync(0xffffffffu, ty, 2);
            if ((l & 3) == 0 && r < R) {
                const float l2 = log2f(sum);
                m_sh[r] = m;
                l_sh[r] = l2;
                w_sh[r] = (ty - m) - l2 * LN2;
            }
        }
    }
    __syncthreads();
    // the logmeanexp over each image's samples and the weights, in double: one warp per image
    const double ln_s = log((double)S);
    double ll_acc = 0.0;
    for (int ii = warp; ii < nimg; ii += MX_THREADS / 32) {
        const long long y = a.labels[img0 + ii];
        const bool ok = y >= 0 && y < C;
        float* lp = w_sh + ii * S;
        double M = -INFINITY;
        for (int s = l; s < S; s += 32) M = fmax(M, (double)lp[s]);
        M = sc_warp_max(M);
        double Q = 0.0;
        for (int s = l; s < S; s += 32) Q += exp((double)lp[s] - M);
        Q = warp_sum(Q);
        __syncwarp();
        for (int s = l; s < S; s += 32) lp[s] = ok ? (float)(exp((double)lp[s] - M) / Q) : 0.0f;
        ll_acc += ok ? M + log(Q) - ln_s : sc_nan();
    }
    if (l == 0) ll_sh[warp] = ll_acc;
    // sweep 2: G and the gradient
    float gw[2][2][32];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int q = 0; q < 32; ++q) gw[mt][nt][q] = 0.0f;
    double gb_acc = 0.0;                                            // thread t: db_t
    for (int tt = 0; tt < tiles; ++tt) {
        __syncthreads();
        load_tile(tt, true);
        float d0[32], d1[32];
        forward(d0, d1);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int rl = 16 * warp + (l >> 2) + 8 * hr, r = tt * MX_TM + rl;
            const long long y = label_of(r);
            const bool in = r < R;
            const float m = in ? m_sh[r] : 0.0f, l2 = in ? l_sh[r] : 0.0f, w = in ? w_sh[r] : 0.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 64 * h + 8 * jj + 2 * (l & 3) + e;
                        const float v = (h ? d1 : d0)[4 * jj + 2 * hr + e] + b_sh[c];
                        const float p = ex2_ftz((v - m) * L2E - l2);
                        const float g = (in && c < C) ? w * ((c == y ? 1.0f : 0.0f) - p) : 0.0f;
                        *reinterpret_cast<uint32_t*>(gt_g + mx_off(MX_N, c, rl)) = to_tf32(g);
                    }
        }
        fence_proxy_async();
        __syncthreads();
        if (t < C)
            for (int rr = 0; rr < MX_TM; ++rr) gb_acc += (double)*reinterpret_cast<const float*>(gt_g + mx_off(MX_N, t, rr));
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < MX_TM / 8; ++ks)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const uint64_t da = make_smem_desc(gt_op + (uint32_t)ks * 2u * MX_N * 16u + (uint32_t)mt * 64u * 16u,
                                                       MX_N * 16, 128);
                    const uint64_t db = make_smem_desc(zt_op + (uint32_t)ks * 2u * MX_N * 16u + (uint32_t)nt * 64u * 16u,
                                                       MX_N * 16, 128);
                    wgmma_m64n64k8_tf32(gw[mt][nt], da, db, 1u);
                }
        wgmma_commit();
        wgmma_wait<0>();
    }
    __syncthreads();
    const int P = nw + C;
    double* part = a.partials + (size_t)blockIdx.x * (P + 1);
    if (t == 0) {
        double s0 = 0.0;
        for (int w = 0; w < MX_THREADS / 32; ++w) s0 += ll_sh[w];
        part[0] = s0;
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int j = 64 * mt + 16 * warp + (l >> 2) + 8 * hr, k = 64 * nt + 8 * jj + 2 * (l & 3) + e;
                        if (j < C && k < C) part[1 + j * C + k] = (double)gw[mt][nt][4 * jj + 2 * hr + e];
                    }
    if (t < C) part[1 + nw + t] = gb_acc;
    __threadfence();
    __syncthreads();
    if (t == 0) last_sh = atomicAdd(a.arrive, 1u) == gridDim.x - 1u;
    __syncthreads();
    if (!last_sh) return;
    __threadfence();
    sc_finish(a, reinterpret_cast<double*>(gb), MX_THREADS, n_img, poisoned);   // (tot over the operands and stats)
}

}  // namespace bbb
