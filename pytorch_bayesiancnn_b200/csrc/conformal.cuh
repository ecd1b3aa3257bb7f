// Split conformal prediction behind the Monte-Carlo step (bbb_mc_conformal_log): appends, for each image of a batch,
// the conformity score of its label (calibration) and the prediction set at a threshold q_hat (prediction) to a
// data-set-long log, at the score log's device-resident cursor (log_claim, score_log.cuh).  A captured step appends
// without a host read, and reads q_hat from device memory, so a threshold set after capture is used by the next replay.
//
// Definitions, image b of a launch at log index i (include/bbb_b200.h states the same):
//   p_c   = exp((double) log_outputs[b, c])  (the exchange's log p_bar)
//   order: classes by log_outputs descending, ties to the smaller class index, -inf last; o(c) = 0-based position of
//          c, S_c = sum of p over the classes before c (double)
//   u     = (r.x + 0.5) * 2^-32, r = philox4x32_10(counter = (i_lo, i_hi, stream_lo, stream_hi), key = seed)
//   E_c   = LAC:  1 - p_c
//           APS:  S_c + u p_c   (randomized; S_c + p_c otherwise)                    Romano et al. 2020
//           RAPS: the APS score + lam * max(0, o(c) + 1 - k_reg)                     Angelopoulos et al. 2021
//   A row that holds a NaN has E_c = NaN for every c (no class is in its set).
//   score[i] = E_y (NaN without a label);  sets[i] bit c = E_c <= q_hat_(c);  size[i] = |set|;  covered[i] = y in set.
//
// INVARIANT (what the coverage guarantee rests on): calibration scores and prediction sets come from one function,
// cf_score, on the same sorted row.  A calibration image re-scored against q_hat is in its own set exactly when its
// logged score is <= q_hat.
//
// One warp per image, grid-stride over the batch.  The warp stages its row in shared memory as 64-bit sort keys
// (~ordered(log p) << 32 | c), sorts them with a bitonic network, takes the prefix sums of p over lane-contiguous
// chunks of the sorted row, and sets the bits of the classes in the set in a shared bit row that lane l writes out as
// word l.
#pragma once
#include "common.cuh"
#include "score_log.cuh"   // log_claim

namespace bbb {

constexpr int CF_MAX_WARPS = 8, CF_MAX_CTAS = 1024;
constexpr int CF_MAX_CLASSES = BBB_CONFORMAL_MAX_CLASSES, CF_WORDS = CF_MAX_CLASSES / 32;
static_assert(CF_WORDS <= 32, "a lane writes one set word");

struct ConformalArgs {
    const float* log_outputs;                   // [B, C]
    const long long* labels;                    // [B], nullable
    int B, C, n_sort, method, randomized, k_reg, per_class;
    double lam;
    uint32_t seed_lo, seed_hi, stream_lo, stream_hi;
    const double* qhat;                         // [1] or [C] (per_class)
    double* score; int* size; int* covered; int* label; unsigned* sets;   // [capacity] x4, [capacity][ceil(C/32)]
    long long capacity;
    unsigned long long* cursor;                 // [2]: next index, images dropped
};

// The conformity score of a class at sorted position pos, p its probability, S the sum of p before it.  The ONE
// definition both the calibration score and the prediction set use (see the invariant above).
__device__ __forceinline__ double cf_score(int method, int randomized, double lam, int k_reg, double u, double S,
                                           double p, int pos) {
    if (method == BBB_CONFORMAL_LAC) return 1.0 - p;
    double e = S + (randomized ? u * p : p);
    if (method == BBB_CONFORMAL_RAPS) e += lam * (double)max(0, pos + 1 - k_reg);
    return e;
}

// float -> key half that sorts ascending as the float sorts descending (-0 as +0; -inf after every finite value)
__device__ __forceinline__ unsigned long long cf_key(float v, int c) {
    if (v == 0.0f) v = 0.0f;
    const uint32_t b = __float_as_uint(v);
    const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((unsigned long long)(~ord) << 32) | (unsigned)c;
}
__device__ __forceinline__ float cf_key_value(unsigned long long k) {
    const uint32_t ord = ~(uint32_t)(k >> 32);
    return __uint_as_float((ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord);
}

// Dynamic shared memory: per warp n_sort keys (8 bytes) and CF_WORDS set words.
__global__ void
conformal_log_kernel(const ConformalArgs a) {
    extern __shared__ __align__(16) unsigned char cf_smem[];
    __shared__ unsigned long long base_sh;
    if (threadIdx.x == 0) log_claim(a.cursor, a.capacity, a.B, base_sh);
    __syncthreads();
    const unsigned long long base = base_sh;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5, n = a.n_sort;
    unsigned long long* keys = (unsigned long long*)cf_smem + (size_t)warp * n;
    unsigned* bits = (unsigned*)((unsigned long long*)cf_smem + (size_t)nwarp * n) + warp * CF_WORDS;
    const int words = (a.C + 31) >> 5, chunk = n >> 5;
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    for (int b = blockIdx.x * nwarp + warp; b < a.B; b += gridDim.x * nwarp) {
        const unsigned long long i = base + (unsigned long long)b;
        if (i >= (unsigned long long)a.capacity) break;          // rows only grow with b
        const float* lo = a.log_outputs + (size_t)b * a.C;
        bool nan_row = false;
        for (int c = lane; c < n; c += 32) {
            const float v = c < a.C ? lo[c] : 0.0f;
            nan_row |= v != v;
            keys[c] = c < a.C ? cf_key(v, c) : ~0ull;              // padding sorts behind every class
        }
        if (lane < CF_WORDS) bits[lane] = 0u;
        nan_row = __any_sync(0xffffffffu, nan_row);
        long long y = a.labels ? a.labels[b] : -1;
        if (y < 0 || y >= a.C) y = -1;                           // a label outside [0, C) counts as none
        // the threshold: NaN anywhere = none yet
        bool no_q = false;
        for (int c = lane; c < (a.per_class ? a.C : 1); c += 32) no_q |= a.qhat[c] != a.qhat[c];
        no_q = __any_sync(0xffffffffu, no_q);
        __syncwarp();
        // bitonic sort, ascending keys = descending log p, ties to the smaller class
        for (int k = 2; k <= n; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int t = lane; t < n; t += 32) {
                    const int p = t ^ j;
                    if (p > t) {
                        const unsigned long long x = keys[t], z = keys[p];
                        if ((x > z) == ((t & k) == 0)) { keys[t] = z; keys[p] = x; }
                    }
                }
                __syncwarp();
            }
        // S before this lane's chunk: the chunk sums, exclusive-scanned over the lanes
        const int p0 = lane * chunk;
        double own = 0.0;
        for (int t = 0; t < chunk; ++t) {
            const unsigned long long k = keys[p0 + t];
            if (p0 + t < a.C) own += exp((double)cf_key_value(k));
        }
        double S = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double v = __shfl_up_sync(0xffffffffu, S, o);
            if (lane >= o) S += v;
        }
        S -= own;
        double u = 1.0;
        if (a.randomized && a.method != BBB_CONFORMAL_LAC) {
            const uint4 r = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), a.stream_lo, a.stream_hi),
                                          make_uint2(a.seed_lo, a.seed_hi));
            u = ((double)r.x + 0.5) * 2.3283064365386963e-10;
        }
        for (int t = 0; t < chunk && p0 + t < a.C; ++t) {
            const unsigned long long k = keys[p0 + t];
            const int c = (int)(unsigned)k;
            const double p = exp((double)cf_key_value(k));
            const double e = nan_row ? qnan : cf_score(a.method, a.randomized, a.lam, a.k_reg, u, S, p, p0 + t);
            S += p;
            if (c == y) a.score[i] = e;
            if (!no_q && e <= a.qhat[a.per_class ? c : 0]) atomicOr(&bits[c >> 5], 1u << (c & 31));
        }
        __syncwarp();
        const unsigned w = lane < words ? bits[lane] : 0u;
        const int sz = __reduce_add_sync(0xffffffffu, __popc(w));
        if (lane < words) a.sets[i * (unsigned long long)words + lane] = no_q ? 0u : w;
        if (lane == 0) {
            if (y < 0) a.score[i] = qnan;
            a.label[i] = (int)y;
            a.size[i] = no_q ? -1 : sz;
            a.covered[i] = (no_q || y < 0) ? -1 : (int)((bits[y >> 5] >> (y & 31)) & 1u);
        }
        __syncwarp();                                             // the next row overwrites keys and bits
    }
}

}  // namespace bbb
