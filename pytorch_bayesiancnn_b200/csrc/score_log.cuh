// Per-image score log of the Monte-Carlo step (bbb_mc_score_log): appends what one exchange produced for each image of a
// batch -- confidence, entropy, mutual information, expected entropy, summed epistemic variance, correctness and the
// predicted class -- to a data-set-long log, at a cursor that lives on the device.  A captured step appends without a
// host read, so steps in flight keep appending in launch order and the host reads the whole log once per data set
// (out-of-distribution detection, selective prediction: uncertainty_estimation.py:61-102 over a whole data set).
//
// Log layout (include/bbb_b200.h): planes[k * capacity + i], k < SL_PLANES, and pred[i]; cursor[0] = next index,
// cursor[1] = images that did not fit.
#pragma once
#include "common.cuh"

namespace bbb {

constexpr int SL_THREADS = 256, SL_MAX_CTAS = 1024, SL_PLANES = 6;
// cursor[0] carries the arrival count of the CTAs of a launch in its top bits while the launch runs (see the kernel)
constexpr int SL_ARRIVE_SHIFT = 48;
constexpr unsigned long long SL_INDEX_MASK = (1ull << SL_ARRIVE_SHIFT) - 1ull;

struct ScoreLogArgs {
    const float* log_outputs;                   // [B, C]
    const float* entropy; const float* expected_entropy; const float* mutual_info;   // [B] each, nullable
    const float* epistemic;                     // [B, C], nullable
    const long long* labels;                    // [B], nullable
    int B, C;
    float* planes; int* pred;                   // [SL_PLANES][capacity], [capacity]
    long long capacity;
    unsigned long long* cursor;                 // [2]: next index, images dropped
};

// The cursor claim of one CTA of a log launch (thread 0 of each CTA; B entries per launch).  The protocol needs no
// counter of its own: every CTA takes the old index into base_sh and counts itself in with ONE atomicAdd of 1 << 48 on
// cursor[0] (index in the low 48 bits, arrivals in the high 16).  The CTA that arrives last has seen every other CTA's
// read, so it alone writes the advanced index (with the arrival bits cleared) and the dropped count; a launch that
// follows in stream order sees both.  Shared by the score log and the probability bank (batchbald.cuh).
__device__ __forceinline__ void log_claim(unsigned long long* cursor, long long capacity, int B,
                                          unsigned long long& base_sh) {
    const unsigned long long old = atomicAdd(cursor, 1ull << SL_ARRIVE_SHIFT);
    const unsigned long long base = old & SL_INDEX_MASK;
    base_sh = base;
    if ((old >> SL_ARRIVE_SHIFT) == gridDim.x - 1u) {
        const unsigned long long cap = (unsigned long long)capacity;
        const unsigned long long fit = base >= cap ? 0ull : min(cap - base, (unsigned long long)B);
        atomicExch(cursor, base + (unsigned long long)B);
        cursor[1] += (unsigned long long)B - fit;
    }
}

// One warp per image, grid-stride over the batch; the cursor as log_claim says.
__global__ void __launch_bounds__(SL_THREADS)
mc_score_log_kernel(const ScoreLogArgs a) {
    __shared__ unsigned long long base_sh;
    if (threadIdx.x == 0) log_claim(a.cursor, a.capacity, a.B, base_sh);
    __syncthreads();
    const unsigned long long base = base_sh;
    const int lane = threadIdx.x & 31, nwarp = SL_THREADS / 32;
    const float qnan = __int_as_float(0x7fffffff);
    for (int b = blockIdx.x * nwarp + (threadIdx.x >> 5); b < a.B; b += gridDim.x * nwarp) {
        const unsigned long long i = base + (unsigned long long)b;
        if (i >= (unsigned long long)a.capacity) break;          // rows only grow with b: the rest of this warp's rows
        const float* lo = a.log_outputs + (size_t)b * a.C;        // fall behind the end too
        // argmax = the first maximal class; -inf ties like any value (a row of -inf gives class 0), NaN is never maximal
        float best = -INFINITY;
        int best_c = 0x7fffffff;
        double epi = 0.0;
        for (int c = lane; c < a.C; c += 32) {
            const float v = lo[c];
            if (v > best || (v == best && c < best_c)) { best = v; best_c = c; }
            if (a.epistemic) epi += (double)a.epistemic[(size_t)b * a.C + c];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
            if (ob > best || (ob == best && oc < best_c)) { best = ob; best_c = oc; }
        }
        if (a.epistemic) epi = warp_sum(epi);
        if (lane == 0) {
            const int pr = best_c == 0x7fffffff ? 0 : best_c;    // every class NaN
            const size_t cap = (size_t)a.capacity;
            float* pl = a.planes + i;
            pl[0] = expf(best);
            pl[cap] = a.entropy ? a.entropy[b] : qnan;
            pl[2 * cap] = a.mutual_info ? a.mutual_info[b] : qnan;
            pl[3 * cap] = a.expected_entropy ? a.expected_entropy[b] : qnan;
            pl[4 * cap] = a.epistemic ? (float)epi : qnan;
            pl[5 * cap] = a.labels ? (a.labels[b] == (long long)pr ? 1.0f : 0.0f) : qnan;
            a.pred[i] = pr;
        }
    }
}

}  // namespace bbb
