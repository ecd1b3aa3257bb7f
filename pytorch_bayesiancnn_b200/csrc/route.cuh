// Routing between task experts (bbb_mc_route): each image goes to the expert that is least uncertain about it, as the
// reference's Split-MNIST mixture does for two experts (Mixtures/utils_mixture.py:119-187,
// predict_using_uncertainty_separate_models / predict_using_confidence_separate_models).  The kernel reads the planes the
// K experts' exchanges wrote, so it runs behind them; it never changes what an expert computes.
//
// Definitions, image b, expert e (include/bbb_b200.h states the same), in double from the fp32 planes:
//   score  EPISTEMIC   sum_c epistemic_e[b, c]           (utils_mixture.py:137-139)
//          ALEATORIC   sum_c aleatoric_e[b, c]           (:140-142)
//          BOTH        sum_c epistemic + sum_c aleatoric (:143-145)
//          MUTUAL_INFO mutual_info_e[b]
//          CONFIDENCE  -exp(max_c log_outputs_e[b, c]); NaN when the row holds a NaN   (:178, on p_bar)
//   e*     the smallest score; ties go to the HIGHEST index (for K = 2 exactly `u2 > u1` of :152 and `max1 > max2` of
//          :178); a NaN score is never chosen while any expert's score is a number (all NaN: e* = K - 1)
//   local  argmax_c pred_e*[b, c], the first maximal class, NaN never maximal (a row of NaN gives 0)   (:154)
//   pred   offset[e*] + local
//
// One warp per image, grid-stride over the batch.  Lane e < K sums expert e's row serially, so a score does not depend
// on the launch shape; the argmin and argmax are comparisons under a total order.  The accumulator's sums are taken per
// warp (in image order), per CTA (in warp order) and over the CTAs (in index order) by the CTA that arrives last; the
// grid is a function of B alone, so equal inputs give equal accumulator bits.
#pragma once
#include "common.cuh"
#include "score_log.cuh"   // log_claim

namespace bbb {

constexpr int RT_THREADS = 256, RT_WARPS = RT_THREADS / 32, RT_MAX_CTAS = 128;
constexpr int RT_MAX_EXPERTS = BBB_ROUTE_MAX_EXPERTS;
// Accumulator, float64 words (bbb_mc_route_bytes): [0] steps [1] images [2] sum_steps local_correct_step / B
// [3] global correct [4] routed to own task [5] invalid labels [RT_SEL + e] images sent to e [RT_SUM + e] sum of e's
// score; word RT_COUNTER holds the CTAs' arrival count (uint32) while a launch runs; behind RT_SCRATCH the per-CTA
// partials [RT_MAX_CTAS][RT_PART]: [0] local correct [1] global correct [2] own task [3] invalid [4 + e] sent to e
// [4 + RT_MAX_EXPERTS + e] score sum of e.
constexpr int RT_SEL = 6, RT_SUM = RT_SEL + RT_MAX_EXPERTS, RT_COUNTER = RT_SUM + RT_MAX_EXPERTS, RT_SCRATCH = RT_COUNTER + 2;
constexpr int RT_PART = 4 + 2 * RT_MAX_EXPERTS;
static_assert(RT_PART <= RT_THREADS, "a thread reduces one partial");
__host__ __device__ inline size_t rt_acc_bytes() { return ((size_t)RT_SCRATCH + (size_t)RT_MAX_CTAS * RT_PART) * sizeof(double); }

struct RouteArgs {
    bbb_route_expert ex[RT_MAX_EXPERTS];        // [B, C] planes (mutual_info [B]) of each expert's exchange
    int offset[RT_MAX_EXPERTS];
    int K, B, C, score, task;
    const long long* labels;                    // [B], nullable
    int* expert; int* local; int* pred; float* scores;   // [B], [B], [B], [B, K]; each nullable
    double* acc;                                // nullable (needs labels)
    int* log_expert; int* log_local; int* log_pred; float* log_scores;   // [capacity] x3, [capacity][K]
    long long capacity;
    unsigned long long* cursor;                 // [2], nullable = no log
};

__device__ __forceinline__ double rt_row_sum(const float* p, int C) {
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += (double)p[c];
    return s;
}

// Expert e's score of image b (lane e of the image's warp), in double; the class sums run in class order.
__device__ __forceinline__ double rt_score(const RouteArgs& a, int e, int b) {
    const bbb_route_expert& x = a.ex[e];
    const size_t row = (size_t)b * a.C;
    switch (a.score) {
    case BBB_ROUTE_EPISTEMIC: return rt_row_sum(x.epistemic + row, a.C);
    case BBB_ROUTE_ALEATORIC: return rt_row_sum(x.aleatoric + row, a.C);
    case BBB_ROUTE_BOTH: return rt_row_sum(x.epistemic + row, a.C) + rt_row_sum(x.aleatoric + row, a.C);
    case BBB_ROUTE_MUTUAL_INFO: return (double)x.mutual_info[b];
    default: {                                                   // BBB_ROUTE_CONFIDENCE
        float m = -INFINITY;
        bool nan = false;
        for (int c = 0; c < a.C; ++c) {
            const float v = x.log_outputs[row + c];
            nan |= v != v;
            m = fmaxf(m, v);
        }
        return nan ? __longlong_as_double(0x7ff8000000000000ll) : -exp((double)m);
    }
    }
}

// (s, e) preferred over (t, f): a number over NaN, then the smaller score, then the higher index -- a total order, so
// the warp's argmin does not depend on the order of the comparisons.
__device__ __forceinline__ bool rt_better(double s, int e, double t, int f) {
    const bool sn = s != s, tn = t != t;
    if (sn != tn) return tn;
    if (!sn && s != t) return s < t;
    return e > f;
}

__global__ void __launch_bounds__(RT_THREADS)
mc_route_kernel(const RouteArgs a) {
    __shared__ unsigned long long base_sh;
    __shared__ double part_sh[RT_WARPS][RT_PART];
    __shared__ unsigned last_sh;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (a.cursor && threadIdx.x == 0) log_claim(a.cursor, a.capacity, a.B, base_sh);
    __syncthreads();
    const unsigned long long base = a.cursor ? base_sh : 0ull;
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    // this warp's sums: lane 0 the four label counts, lane e < K expert e's count and score sum
    double n_local = 0.0, n_global = 0.0, n_own = 0.0, n_bad = 0.0, n_sel = 0.0, s_sum = 0.0;
    for (int b = blockIdx.x * RT_WARPS + warp; b < a.B; b += gridDim.x * RT_WARPS) {
        const double s = lane < a.K ? rt_score(a, lane, b) : qnan;
        double bs = s;
        int be = lane < a.K ? lane : -1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double os = __shfl_xor_sync(0xffffffffu, bs, o);
            const int oe = __shfl_xor_sync(0xffffffffu, be, o);
            if (oe >= 0 && (be < 0 || rt_better(os, oe, bs, be))) { bs = os; be = oe; }
        }
        const int es = be;                                        // every lane holds e*
        const float* pr = a.ex[es].pred + (size_t)b * a.C;
        float best = -INFINITY;
        int best_c = 0x7fffffff;
        for (int c = lane; c < a.C; c += 32) {
            const float v = pr[c];
            if (v > best || (v == best && c < best_c)) { best = v; best_c = c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
            if (ob > best || (ob == best && oc < best_c)) { best = ob; best_c = oc; }
        }
        const int loc = best_c == 0x7fffffff ? 0 : best_c;
        const int gp = a.offset[es] + loc;
        if (lane < a.K) {
            if (a.scores) a.scores[(size_t)b * a.K + lane] = (float)s;
            n_sel += lane == es ? 1.0 : 0.0;
            s_sum += s;
        }
        if (lane == 0) {
            if (a.expert) a.expert[b] = es;
            if (a.local) a.local[b] = loc;
            if (a.pred) a.pred[b] = gp;
            if (a.labels) {
                // the label's task and its local and global class; a label no range holds is invalid (counted wrong)
                const long long y = a.labels[b];
                int tk = -1;
                long long ly = -1, gy = -1;
                if (a.task >= 0) {
                    if (y >= 0 && y < a.C) { tk = a.task; ly = y; gy = a.offset[a.task] + y; }
                } else {
                    for (int e = 0; e < a.K && tk < 0; ++e)
                        if (y >= a.offset[e] && y < (long long)a.offset[e] + a.C) { tk = e; ly = y - a.offset[e]; gy = y; }
                }
                n_bad += tk < 0 ? 1.0 : 0.0;
                n_local += (tk >= 0 && ly == loc) ? 1.0 : 0.0;
                n_global += (tk >= 0 && gy == gp) ? 1.0 : 0.0;
                n_own += (tk >= 0 && tk == es) ? 1.0 : 0.0;
            }
        }
        if (a.cursor) {
            const unsigned long long i = base + (unsigned long long)b;
            if (i < (unsigned long long)a.capacity) {
                if (lane < a.K) a.log_scores[i * (unsigned long long)a.K + lane] = (float)s;
                if (lane == 0) { a.log_expert[i] = es; a.log_local[i] = loc; a.log_pred[i] = gp; }
            }
        }
    }
    if (!a.acc) return;
    if (lane == 0) {
        part_sh[warp][0] = n_local; part_sh[warp][1] = n_global; part_sh[warp][2] = n_own; part_sh[warp][3] = n_bad;
    }
    if (lane < RT_MAX_EXPERTS) {
        part_sh[warp][4 + lane] = lane < a.K ? n_sel : 0.0;
        part_sh[warp][4 + RT_MAX_EXPERTS + lane] = lane < a.K ? s_sum : 0.0;
    }
    __syncthreads();
    unsigned* counter = reinterpret_cast<unsigned*>(a.acc + RT_COUNTER);
    if (threadIdx.x < RT_PART) {                                  // this CTA's partials, its warps in order
        double v = 0.0;
        for (int w = 0; w < RT_WARPS; ++w) v += part_sh[w][threadIdx.x];
        a.acc[RT_SCRATCH + (size_t)blockIdx.x * RT_PART + threadIdx.x] = v;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(counter, 1u);
        last_sh = prev == gridDim.x - 1;
    }
    __syncthreads();
    if (!last_sh) return;
    __threadfence();                                              // the other CTAs' partials, read below
    if (threadIdx.x < RT_PART) {
        double v = 0.0;
        for (unsigned i = 0; i < gridDim.x; ++i) v += __ldcg(a.acc + RT_SCRATCH + (size_t)i * RT_PART + threadIdx.x);
        const int t = threadIdx.x;
        if (t == 0) a.acc[2] += v / (double)a.B;                   // the batch's local accuracy (np.mean(accs) sums these)
        else if (t < 4) a.acc[2 + t] += v;
        else if (t < 4 + RT_MAX_EXPERTS) { if (t - 4 < a.K) a.acc[RT_SEL + t - 4] += v; }
        else if (t - 4 - RT_MAX_EXPERTS < a.K) a.acc[RT_SUM + t - 4 - RT_MAX_EXPERTS] += v;
    }
    if (threadIdx.x == 0) {
        a.acc[0] += 1.0;
        a.acc[1] += (double)a.B;
        *counter = 0u;
    }
}

}  // namespace bbb
