// Temperature scaling of the Monte-Carlo predictive (Guo et al. 2017), applied per sample before the softmax and the
// average over samples, as for MC-dropout nets (Laves et al. 2019):  p_bar_T = mean_s softmax(z_s / T)
// (include/bbb_b200.h, bbb_mc_logit_log / bbb_temperature_nll / bbb_mc_temper):
//
//  (L) mc_logit_log_kernel    -- appends one step's raw per-sample logits and its labels to a calibration bank, at the
//      score log's device-resident cursor (log_claim, score_log.cuh).  Bank layout: bank[i][s][c] fp32, labels[i] int64.
//  (F) temperature_nll_kernel -- the bank's mean NLL of the tempered predictive at K temperatures in one launch:
//          l(T) = -(1/n) sum_i log( (1/S) sum_s softmax(z_is / T)[y_i] )
//      One warp per image, one lane per sample row (s = lane, lane + 32, ..): a lane reads its row 2 ceil(K / 11) times,
//      a max pass and an exponential pass per sweep of 11 temperatures (the accumulators one sweep keeps in registers);
//      after the first pass the reads hit L1 / L2.  The lanes' loads are C floats apart (not coalesced), and lanes
//      s >= S idle: with S < 32 only S of 32 lanes work.
//      One CTA per fixed block of TN_CTA_IMAGES images (a function of the image index alone); per-image terms summed in
//      double per warp, per CTA and over the CTAs in index order by the last CTA to arrive, so the result does not
//      depend on the launch's grid.  That CTA also takes the argmin and writes the next search round's grid.
//  (T) mc_temper_kernel       -- z <- z / T in place on a step's logits, T read from device memory at run time.
#pragma once
#include "common.cuh"
#include "fwd_tc.cuh"      // pdl_wait / pdl_trigger
#include "score_log.cuh"   // log_claim

namespace bbb {

// ---- (L) logit bank -------------------------------------------------------------------------------------------
constexpr int LL_THREADS = 256, LL_MAX_CTAS = 1024;

struct LogitLogArgs {
    const float* logits;                        // [S, B, C]: the step's per-sample logits
    const long long* labels;                    // [B], nullable: -1 is logged
    int S, B, C;
    float* bank; long long* bank_labels;        // [capacity][S][C], [capacity]
    long long capacity;
    unsigned long long* cursor;                 // [2]: next index, images dropped
};

// One CTA per image (grid-stride over the batch); the image's S rows of C land contiguously in its entry.
__global__ void __launch_bounds__(LL_THREADS)
mc_logit_log_kernel(const LogitLogArgs a) {
    __shared__ unsigned long long base_sh;
    if (threadIdx.x == 0) log_claim(a.cursor, a.capacity, a.B, base_sh);
    __syncthreads();
    const unsigned long long base = base_sh;
    const int row = a.S * a.C;
    for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
        const unsigned long long i = base + (unsigned long long)b;
        if (i >= (unsigned long long)a.capacity) break;          // entries only grow with b
        float* dst = a.bank + (size_t)i * row;
        for (int r = threadIdx.x; r < row; r += LL_THREADS) {
            const int s = r / a.C, c = r - s * a.C;
            dst[r] = a.logits[((size_t)s * a.B + b) * a.C + c];
        }
        if (threadIdx.x == 0) a.bank_labels[i] = a.labels ? a.labels[b] : -1ll;
    }
}

// ---- (F) NLL at K temperatures, and the search between passes ---------------------------------------------------
constexpr int TN_THREADS = 256, TN_WARPS = TN_THREADS / 32;
constexpr int TN_IMAGES = 4;                                   // images per warp
constexpr int TN_CTA_IMAGES = TN_WARPS * TN_IMAGES;            // images per CTA
constexpr int TN_MAX_K = 64;                                   // temperatures per pass
static_assert(TN_CTA_IMAGES == BBB_TEMPERATURE_CTA_IMAGES && TN_MAX_K == BBB_TEMPERATURE_MAX_POINTS,
              "temperature fit: header and kernel disagree");
constexpr int TN_KC = 11;                                      // temperatures per row sweep (register accumulators;
                                                               // 3 x 11 = the default search's 32 points and T = 1)

struct TempNllArgs {
    const float* logits;                        // [n][S][C]
    const long long* labels;                    // [n]
    const long long* cursor;                    // nullable: images = min(cursor[0], n); cursor[1] > 0 poisons
    int n, S, C, K, K_search, first, last;
    const double* tau;                          // [K]: ln T
    double* nll;                                // [K]
    double* next_tau;                           // [K_search], nullable
    double* fit;                                // [4]: nll at T = 1, nll, at_bound, tau of the result
    float* temperature;                         // [1], written by the last pass
    double* partials;                           // [gridDim.x][K]
    unsigned int* arrive;                       // zero between launches (the last CTA resets it)
};

// Equally spaced points on [lo, hi], each rounded as lo + ((hi - lo) * k) / (K - 1) is in IEEE double (the host
// planner mc.temperature_grid forms round 0 the same way).
__device__ __forceinline__ double tn_point(double lo, double hi, int k, int K) {
    return __dadd_rn(lo, __ddiv_rn(__dmul_rn(__dsub_rn(hi, lo), (double)k), (double)(K - 1)));
}

// 2^x by one MUFU.EX2 (2 ulp; results below 2^-126 flush to 0, which no sum that holds a term >= 1 can see)
__device__ __forceinline__ float ex2_ftz(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Per (i, s): d_c = z_c - max_c z (fp32), log2 p_s[y] = d_y a_k - log2 sum_c exp2(d_c a_k), a_k = log2(e) / T_k in fp32
// (ex2_ftz / accurate log2f); the logmeanexp over s is an online (max, sum) in fp32 per lane and then across the
// warp; the image's term ((max + log2 sum) ln 2 - ln S) and every sum after it are double.
__global__ void __launch_bounds__(TN_THREADS)
temperature_nll_kernel(const TempNllArgs a) {
    __shared__ float a2_sh[TN_MAX_K + TN_KC];
    __shared__ double part_sh[TN_WARPS][TN_MAX_K];
    __shared__ int last_sh;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < TN_MAX_K + TN_KC)
        a2_sh[threadIdx.x] = threadIdx.x < a.K ? (float)(exp(-a.tau[threadIdx.x]) * 1.4426950408889634) : 0.0f;
    long long n_img = a.n;
    bool poisoned = false;
    if (a.cursor) {
        n_img = min(a.cursor[0], (long long)a.n);
        poisoned = a.cursor[1] != 0;
    }
    __syncthreads();
    const int chunks = (a.K + TN_KC - 1) / TN_KC, kc = (a.K + chunks - 1) / chunks;
    double acc_lo = 0.0, acc_hi = 0.0;          // this warp's sums of log-likelihoods at k = lane, lane + 32
    const double ln_s = log((double)a.S), ln2 = 0.6931471805599453;
    for (int j = 0; j < TN_IMAGES; ++j) {
        const long long i = (long long)blockIdx.x * TN_CTA_IMAGES + warp * TN_IMAGES + j;
        if (i >= n_img) break;
        const long long y = a.labels[i];
        const bool ok = y >= 0 && y < a.C;
        const float* img = a.logits + (size_t)i * a.S * a.C;
        for (int k0 = 0; k0 < a.K; k0 += kc) {
            float ak[TN_KC], M[TN_KC], Q[TN_KC];
#pragma unroll
            for (int q = 0; q < TN_KC; ++q) { ak[q] = a2_sh[k0 + q]; M[q] = -INFINITY; Q[q] = 0.0f; }
            for (int s = lane; s < a.S; s += 32) {
                const float* row = img + (size_t)s * a.C;
                float m = -INFINITY;
                for (int c = 0; c < a.C; ++c) m = fmaxf(m, __ldg(row + c));
                float e[TN_KC];
#pragma unroll
                for (int q = 0; q < TN_KC; ++q) e[q] = 0.0f;
                for (int c = 0; c < a.C; ++c) {
                    const float d = __ldg(row + c) - m;
#pragma unroll
                    for (int q = 0; q < TN_KC; ++q) e[q] += ex2_ftz(d * ak[q]);      // (slots q >= kc: unused)
                }
                const float dy = ok ? __ldg(row + y) - m : 0.0f;
#pragma unroll
                for (int q = 0; q < TN_KC; ++q) {
                    const float lp = dy * ak[q] - log2f(e[q]);
                    if (lp > M[q]) { Q[q] = Q[q] * ex2_ftz(M[q] - lp) + 1.0f; M[q] = lp; }
                    else Q[q] += ex2_ftz(lp - M[q]);
                }
            }
#pragma unroll
            for (int q = 0; q < TN_KC; ++q) {
                float m = M[q], t = Q[q];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), t2 = __shfl_xor_sync(0xffffffffu, t, o);
                    const float mn = fmaxf(m, m2);
                    t = (m == -INFINITY ? 0.0f : t * ex2_ftz(m - mn)) + (m2 == -INFINITY ? 0.0f : t2 * ex2_ftz(m2 - mn));
                    m = mn;
                }
                const int k = k0 + q;
                if (q < kc && k < a.K && (k == lane || k == lane + 32)) {
                    const double ll = ok ? ((double)m + log2((double)t)) * ln2 - ln_s : nan("");
                    if (k == lane) acc_lo += ll; else acc_hi += ll;
                }
            }
        }
    }
    if (lane < a.K) part_sh[warp][lane] = acc_lo;
    if (lane + 32 < a.K) part_sh[warp][lane + 32] = acc_hi;
    __syncthreads();
    if (threadIdx.x < a.K) {
        double t = 0.0;
        for (int w = 0; w < TN_WARPS; ++w) t += part_sh[w][threadIdx.x];
        a.partials[(size_t)blockIdx.x * a.K + threadIdx.x] = t;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) last_sh = atomicAdd(a.arrive, 1u) == gridDim.x - 1u;
    __syncthreads();
    if (!last_sh) return;
    __threadfence();
    if (threadIdx.x < a.K) {
        double t = 0.0;
#pragma unroll 8
        for (int b = 0; b < (int)gridDim.x; ++b) t += __ldcg(a.partials + (size_t)b * a.K + threadIdx.x);
        a.nll[threadIdx.x] = poisoned ? nan("") : -t / (double)n_img;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    *a.arrive = 0u;
    __threadfence();
    if (a.K_search < 1) return;
    // k* = the first minimal NLL of the search points (a NaN is never minimal; all NaN: 0)
    int ks = 0;
    double best = INFINITY;
    for (int k = 0; k < a.K_search; ++k) {
        const double v = a.nll[k];
        if (v < best) { best = v; ks = k; }
    }
    if (a.first) {
        a.fit[0] = a.K > a.K_search ? a.nll[a.K_search] : nan("");
        a.fit[2] = (ks == 0 || ks == a.K_search - 1) ? 1.0 : 0.0;
    }
    if (a.next_tau) {
        const double lo = a.tau[max(ks - 1, 0)], hi = a.tau[min(ks + 1, a.K_search - 1)];
        for (int k = 0; k < a.K_search; ++k) a.next_tau[k] = tn_point(lo, hi, k, a.K_search);
    }
    if (a.last) {
        const double at_one = a.fit[0], v = a.nll[ks];
        if (isnan(at_one) || isnan(v)) {               // no fit: *temperature keeps the value engines read now
            a.fit[1] = a.fit[3] = nan("");
        } else if (v > at_one) {                 // never worse than T = 1 on the bank
            a.fit[1] = at_one; a.fit[3] = 0.0;
            *a.temperature = 1.0f;
        } else {
            a.fit[1] = v; a.fit[3] = a.tau[ks];
            *a.temperature = (float)exp(a.tau[ks]);
        }
    }
}

// ---- (T) temper ------------------------------------------------------------------------------------------------
constexpr int TP_THREADS = 256, TP_MAX_CTAS = 1024;

// z[j] <- z[j] / *t (IEEE division, the bits of torch's fp32 z / T), float4 over the 16-byte aligned body.  Launched
// with programmatic serialization behind the kernel that writes z: waits for it before reading anything.
__global__ void __launch_bounds__(TP_THREADS)
mc_temper_kernel(float* z, long long n, const float* t) {
    pdl_wait();
    pdl_trigger();
    const float T = *t;
    const long long tid = (long long)blockIdx.x * TP_THREADS + threadIdx.x, stride = (long long)gridDim.x * TP_THREADS;
    const long long head = min((long long)((16u - ((unsigned)(uintptr_t)z & 15u)) & 15u) / 4, n);
    const long long body = (n - head) >> 2, tail0 = head + body * 4;
    float4* v = reinterpret_cast<float4*>(z + head);
    for (long long k = tid; k < body; k += stride) {
        float4 q = v[k];
        q.x = __fdiv_rn(q.x, T); q.y = __fdiv_rn(q.y, T); q.z = __fdiv_rn(q.z, T); q.w = __fdiv_rn(q.w, T);
        v[k] = q;
    }
    if (tid < head) z[tid] = __fdiv_rn(z[tid], T);
    if (tid < n - tail0) z[tail0 + tid] = __fdiv_rn(z[tail0 + tid], T);
}

}  // namespace bbb
