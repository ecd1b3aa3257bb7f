// Monte-Carlo combine + ELBO head + uncertainty outputs, fused with the ONE exchange of the forward path.
//
// What sits directly above the Bayesian layers (SURVEY.md 8e, rows f3/f4):
//   main_bayesian.py:46-53   outputs[:,:,j] = log_softmax(net(x)); log_outputs = logmeanexp_j; kl = mean_j kl_j
//   utils.py:14-22           logmeanexp
//   metrics.py:12-14,23-24   ELBO = nll_loss(log_outputs, y, mean) * train_size + beta * kl ; acc
//   uncertainty_estimation.py:70-96   p_hat = softmax (or softplus-normalised, :73-77); pred = mean_t logits;
//                            epistemic = diag((p_hat - p_bar)^T (p_hat - p_bar)) / T; aleatoric = diag(diag(p_bar) - p_hat^T p_hat / T)
//
// The num_ens samples are sharded over ranks (one process per GPU).  Every rank reduces ITS samples to per-(image,
// class) partials, pushes them straight into every peer's receive buffer over NVLink (plain st.global on peer-mapped
// memory obtained through CUDA IPC), raises a per-CTA flag with release semantics, waits for the peers' flags, and
// finishes the reduction + head locally -- one kernel, no NCCL, no host round trip.  The partials are the exact
// (max, sum-exp) pairs of logmeanexp, so the result equals the reference's logmeanexp even where every sample's
// probability underflows (a plain sum of softmaxes does not).
//
// Receive buffer of one rank (all ranks use the same layout):
//   [0, 4096)                       reserved
//   [4096, ...)                     u64 data[2 slots][world][n_planes * B * C + 2 (+ B with INFO)]
// Per sending rank: the n_planes [B, C] planes, the KL word at n_planes * B * C, a spare word, and -- only in the INFO
// instantiation -- a plane of B words behind them: sum over the rank's samples of H[p_hat_s] per image.
// Row blocks (bbb_mc_exchange_sharded, world = Rs sample groups x Rb row blocks): [2 slots][Rs][...] of the same layout,
// one sender slot per sample group; rank (g, k) writes the words of its rows [b0, b1) into slot g, the group's block-0
// rank also the KL word.  Every row of a slot then comes from exactly one rank of its group.
//
// INFO (BBB_MC_INFO) adds the two other terms of the entropy decomposition H[p_bar] = E_s H[p_hat_s] + I(y; w):
//   H[p]                   = -sum_c p_c log p_c, with 0 log 0 = 0 (a class whose probability underflows adds nothing)
//   expected_entropy[b]    = (1/S_total) sum_{s over all ranks} H[p_hat_s[b]]      (aleatoric)
//   mutual_info[b]         = entropy[b] - expected_entropy[b]  in fp32, not clamped: rounding may leave it slightly < 0
// p_hat_s is the same softmax (or softplus-normalised) row the moments use.
// Every float travels as ONE 8-byte store {value bits, sequence number} (the "LL" idea of NCCL's low-latency protocol):
// 8-byte stores are single-copy atomic over NVLink, so the receiver simply polls each word until its tag equals the
// launch's sequence number -- no fence, no separate flag, no CTA barrier between the push and the finish.  (A fence.sys +
// st.release.sys flag per CTA instead would put two system-scope fences per step on the critical path.)
// Tags make the buffer reusable without a reset: launch k of a rank uses slot k & 1; a peer can be at most one launch
// ahead (it cannot finish launch k+1 before it has OUR launch k+1 words, which we send after we finished reading k).
#pragma once
#include "common.cuh"

namespace bbb {

constexpr int MCX_MAX_RANKS = 16, MCX_MAX_CTAS = 64, MCX_CTRL_BYTES = 4096, MCX_THREADS = 256, MCX_MAX_SLOCAL = 256;

struct McxArgs {
    const float* logits;          // [S_local, B, C] this rank's samples
    const float* kl;              // n_kl device floats whose SUM is the KL of ONE sample (e.g. the per-layer terms; identical for
    int n_kl;                     // every sample, SURVEY D11); nullable
    unsigned long long* noise_base; unsigned long long noise_inc;   // optional: *noise_base += noise_inc when the launch is done
    int S_local, S_total, B, C;
    int want_moments, normalized; // moments: also exchange sum p, sum p^2, sum logits;  normalized: p_hat = softplus/sum softplus
    const long long* labels;      // [B] int64, nullable
    float train_size, beta;
    int rank, world;
    unsigned char* peer[MCX_MAX_RANKS];   // receive buffers; peer[rank] is the local one
    unsigned int* seq;            // local device counter: launches completed so far
    unsigned int* done;           // local device counter (zeroed once): CTAs finished in this launch
    unsigned int* timeouts;       // local device counter: waits that gave up (a peer never delivered) -- results are then invalid
    unsigned long long timeout_ns;
    double* head_partials;        // [MCX_MAX_CTAS][2] nll sum, correct count
    // outputs (local)
    float* log_outputs;           // [B, C]
    float* kl_out;                // scalar: sum_j kl_j / S_total
    float* pred; float* epistemic; float* aleatoric; float* entropy;   // [B,C] x3, [B]; nullable (need want_moments)
    float* head;                  // [4]: loss, nll, accuracy, beta*kl; nullable (needs labels)
    long long* tl;                // debug timeline slot (nullptr in production)
    long long* trace;             // debug: [CTA][8] %globaltimer stamps of the handshake (nullptr in production)
    float* expected_entropy; float* mutual_info;   // [B] each; nullable; written by the INFO instantiation only
    // row blocks (the SHARD instantiation only, bbb_mc_exchange_sharded): this rank is row block `block` of sample group
    // `group` of `groups`; its logits are [S_local, rows, C] for images [row0, row0 + rows); the receive buffer has one
    // slot per group, which the group's row blocks fill together
    int groups, group, block, row0, rows;
    double* metrics;              // the METRICS instantiation only (bbb_mc_exchange_metrics): accumulator + per-CTA scratch
};

// Evaluation accumulator (METRICS, bbb_mc_exchange_metrics), float64 words; every launch adds one step:
//   [0] steps  [1] images  [2] sum_steps nll_step  [3] sum_steps acc_step  [4] sum_steps klsum_step
//   [MCM_HEAD + i] = sum over images of part i, i < MCM_PART:
//     [0] nll  [1] correct  [2] brier  [3 + m] bin count  [3 + BINS + m] bin sum conf  [3 + 2 BINS + m] bin sum correct
// and behind the first MCM_SCRATCH words the per-CTA partials [MCX_MAX_CTAS][MCM_PART] of the launch.
constexpr int MCM_BINS = 15, MCM_HEAD = 5, MCM_PART = 3 + 3 * MCM_BINS, MCM_WORDS = MCM_HEAD + MCM_PART, MCM_SCRATCH = 64;
static_assert(MCM_WORDS <= MCM_SCRATCH, "accumulator overlaps the per-CTA scratch");
static_assert(MCM_PART % 2 == 0 && MCM_PART / 2 <= 32, "a warp carries two parts per lane");
__host__ __device__ inline size_t mcm_bytes() { return ((size_t)MCM_SCRATCH + (size_t)MCX_MAX_CTAS * MCM_PART) * sizeof(double); }
// dynamic shared memory of a launch: the per-warp row normalisers, then (METRICS) the CTA's partials and the last-CTA flag
// (392 bytes: the exchange CTA has to fit beside a GEMM and a prep CTA of the next step, see mc_exchange_kernel)
__host__ inline size_t mcx_smem_bytes(int S_local, bool metrics) {
    return (size_t)(MCX_THREADS / 32) * S_local * sizeof(float) + (metrics ? (size_t)(MCM_PART + 1) * sizeof(double) : 0);
}

__host__ __device__ inline int mcx_planes(int want_moments) { return want_moments ? 5 : 2; }
__host__ __device__ inline size_t mcx_info_off(int B, int C, int want_moments) { return (size_t)mcx_planes(want_moments) * B * C + 2; }
__host__ __device__ inline size_t mcx_rank_floats(int B, int C, int want_moments, bool info = false) {
    return mcx_info_off(B, C, want_moments) + (info ? (size_t)B : 0);
}
__host__ inline size_t mcx_buffer_bytes(int B, int C, int want_moments, int world, bool info = false) {
    return MCX_CTRL_BYTES + 2 * (size_t)world * mcx_rank_floats(B, C, want_moments, info) * sizeof(unsigned long long);
}

__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned int seq) {
    const unsigned long long w = ((unsigned long long)seq << 32) | (unsigned long long)__float_as_uint(v);
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_ll(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float softplus_f(float v) { return v > 20.0f ? v : log1pf(expf(v)); }   // F.softplus(beta=1, threshold=20)

// <= 51 registers: an exchange CTA has to fit beside a GEMM CTA (320 x ~120 registers) and a prep CTA of the next step.
// INFO: also expected_entropy / mutual_info (the extra plane of the receive buffer); INFO == false is the default kernel.
// SHARD: row blocks (bbb_mc_exchange_sharded).  The rank pushes the partials of ITS rows into slot `group` of every peer
// (the group's block-0 rank also its KL word), and every rank finishes all B rows from the `groups` slots, in ascending
// group order -- with groups == world and one block per group that is exactly the default kernel's work.
// METRICS: also add this step to the evaluation accumulator p.metrics (needs labels).  Per image, on p_bar = exp(log_outputs):
// nll, correct (argmax == label), brier = sum_c (p_bar_c - [c == y])^2 and the calibration bin m = clamp(ceil(conf * 15) - 1,
// 0, 14) of conf = p_bar[argmax].  A warp keeps its partials in registers, spread over its lanes (lane l holds parts 2l and
// 2l + 1); the warps add them into the CTA's shared partials in warp order, and the last CTA sums the CTAs in order
// (double throughout, no float atomics): bitwise the same on every rank and every run.  Takes the cross-CTA finish even
// with one rank.
template <bool INFO, bool SHARD = false, bool METRICS = false>
__global__ void __launch_bounds__(MCX_THREADS, 5)
mc_exchange_kernel(const McxArgs p) {
    // per warp: log-sum-exp (or softplus sum) of each local sample's row -- dynamic, 32 * S_local bytes: next to a 193 KB
    // GEMM CTA and a 26 KB prep CTA of the NEXT step (overlap mode) a fixed 8 KB array did not fit on the SM any more
    extern __shared__ float norm_dyn[];
    __shared__ unsigned int seq_sh;
    __shared__ double red[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = MCX_THREADS / 32;
    const int B = p.B, C = p.C, BC = B * C;
    const int rows_per_cta = (B + gridDim.x - 1) / gridDim.x;
    const int b0 = blockIdx.x * rows_per_cta, b1 = min(B, b0 + rows_per_cta);
    tl_enter(p.tl);
    asm volatile("griddepcontrol.wait;" ::: "memory");      // launched with programmatic serialization: the logits come from the predecessor
    tl_dep(p.tl);
    const bool tracer = p.trace && threadIdx.x == (p.rank + 1) % p.world;      // the thread that talks to the next rank
    long long* tr = p.trace + blockIdx.x * 8;
    if (tracer) tr[0] = (long long)globaltimer_ns();
    if (threadIdx.x == 0) seq_sh = *p.seq + 1u;
    double* mcm_cta = reinterpret_cast<double*>(norm_dyn + nwarp * p.S_local);     // METRICS: [MCM_PART]
    if constexpr (METRICS)
        if (threadIdx.x < MCM_PART) mcm_cta[threadIdx.x] = 0.0;
    __syncthreads();
    const unsigned int seq = seq_sh;
    const size_t rank_floats = mcx_rank_floats(B, C, p.want_moments, INFO);
    // senders of one launch: ranks, or sample groups in row-block mode; this rank's partials go to sender slot `src`
    auto nsrc = [&] { return SHARD ? p.groups : p.world; };
    auto src = [&] { return SHARD ? p.group : p.rank; };
    // the images [pb0, pb1) this CTA reduces and pushes: the images it finishes, unless the rank holds a row block
    const int nrows = SHARD ? p.rows : B, rowoff = SHARD ? p.row0 : 0;
    int pb0 = b0, pb1 = b1;
    if constexpr (SHARD) {
        const int rpc = (nrows + gridDim.x - 1) / gridDim.x;
        pb0 = rowoff + blockIdx.x * rpc; pb1 = min(rowoff + nrows, pb0 + rpc);
    }
    const size_t slot_off = (size_t)(seq & 1u) * nsrc() * rank_floats;        // in words, behind the control block
    const float inv_S = 1.0f / (float)p.S_total;

    const unsigned long long* rx = reinterpret_cast<const unsigned long long*>(p.peer[p.rank] + MCX_CTRL_BYTES) + slot_off;
    const bool solo = p.world == 1;     // one rank: the partials never leave the registers (no buffer round trip, no handshake)
    // nll and correct count of the head, on lane 0.  METRICS: lane l < MCM_PART / 2 of a warp sums parts 2l and 2l + 1 of
    // its rows in them (lane 0's are the head's two), so the partials need no registers or shared memory of their own
    double nll_acc = 0.0, hit_acc = 0.0;
    // per-row state of the finish (4): running argmax, entropy, the label's log-probability
    struct RowFin { float best; int best_c; float ent, lab_lp; long long lab; };
    auto fin_elem = [&](RowFin& rf, size_t e, int c, float M, float tot, float sp, float sp2, float sl) {
        const float lo = M + logf(tot * inv_S);                           // utils.py:14-22
        p.log_outputs[e] = lo;
        if (lo > rf.best) { rf.best = lo; rf.best_c = c; }
        if ((long long)c == rf.lab) rf.lab_lp = lo;
        if (p.want_moments) {
            const float pbar = sp * inv_S, p2 = sp2 * inv_S;
            if (p.pred) p.pred[e] = sl * inv_S;                           // uncertainty_estimation.py:82-83
            if (p.epistemic) p.epistemic[e] = p2 - pbar * pbar;           // :89-91  (E[p^2] - p_bar^2)
            if (p.aleatoric) p.aleatoric[e] = pbar - p2;                  // :94-95  (p_bar - E[p^2])
            rf.ent -= pbar > 0.0f ? pbar * logf(pbar) : 0.0f;             // H[p_bar] (no reference, SURVEY D3)
        }
    };
    // row reductions: entropy, the label's log-probability, argmax (first maximal class, like torch.argmax on ties);
    // hsum (INFO): sum over all S_total samples of H[p_hat_s] of this image
    auto fin_row = [&](RowFin& rf, int b, float hsum) {
        float ent = warp_sum(rf.ent), lab_lp = warp_sum(rf.lab_lp), best = rf.best;
        int best_c = rf.best_c;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
            if (ob > best || (ob == best && oc < best_c)) { best = ob; best_c = oc; }
        }
        if constexpr (METRICS) {
            // Brier score from the log_outputs this lane wrote for the row (no extra register state in the class loop);
            // per element (p - [c == y])^2, never the expanded form, which cancels
            double br = 0.0;
            for (int c = lane; c < C; c += 32) {
                const double d = (double)expf(p.log_outputs[(size_t)b * C + c]) - ((long long)c == rf.lab ? 1.0 : 0.0);
                br += d * d;
            }
            br = warp_sum(br);                      // br, lab_lp, best, best_c: the same on every lane
            const float conf = expf(best);
            const int m = min(max((int)ceilf(conf * (float)MCM_BINS) - 1, 0), MCM_BINS - 1);
            const double hit = (best_c == (int)rf.lab) ? 1.0 : 0.0;
            auto part = [&](int i) {                // this row's part i; + 0.0 leaves a sum unchanged
                return i == 0 ? -(double)lab_lp : i == 1 ? hit : i == 2 ? br : i == 3 + m ? 1.0
                     : i == 3 + MCM_BINS + m ? (double)conf : i == 3 + 2 * MCM_BINS + m ? hit : 0.0;
            };
            if (lane > 0 && lane < MCM_PART / 2) { nll_acc += part(2 * lane); hit_acc += part(2 * lane + 1); }
        }
        if (lane == 0) {
            if (p.entropy && p.want_moments) p.entropy[b] = ent;
            if constexpr (INFO) {
                const float ee = __fmul_rn(hsum, inv_S);   // not fused into the subtraction: mutual_info == entropy - ee exactly
                if (p.expected_entropy) p.expected_entropy[b] = ee;
                if (p.mutual_info) p.mutual_info[b] = ent - ee;
            }
            if (p.labels) { nll_acc -= (double)lab_lp; hit_acc += (best_c == (int)rf.lab) ? 1.0 : 0.0; }
        }
    };

    // a word of the receive buffer, once its tag says it belongs to this launch (never hangs: a lost peer = a counted timeout)
    auto ll_value = [&](unsigned long long v, const unsigned long long* w) -> float {
        if ((unsigned int)(v >> 32) != seq) {
            const unsigned long long t0 = globaltimer_ns();
            unsigned int spins = 0;
            while ((unsigned int)((v = ld_ll(w)) >> 32) != seq) {
                __nanosleep(64);          // the SM is shared with the next step's kernels (overlap mode): do not hammer the LSU
                if ((++spins & 63u) == 0u && globaltimer_ns() - t0 > p.timeout_ns) { atomicAdd(p.timeouts, 1u); break; }
            }
        }
        return __uint_as_float((unsigned int)v);
    };

    // ---- (1) local partials of this CTA's images, pushed to every rank's receive buffer ---------------------
    for (int b = pb0 + warp; b < pb1; b += nwarp) {
        const int bl = b - rowoff;                               // local row of image b
        for (int s = 0; s < p.S_local; ++s) {                   // row normaliser of every local sample
            const float* row = p.logits + ((size_t)s * nrows + bl) * C;
            float r;
            if (p.normalized) {
                float acc = 0.0f;
                for (int c = lane; c < C; c += 32) acc += softplus_f(row[c]);
                r = warp_sum(acc);
            } else {
                float mx = -INFINITY;
                for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                float se = 0.0f;
                for (int c = lane; c < C; c += 32) se += expf(row[c] - mx);
                r = mx + logf(warp_sum(se));
            }
            if (lane == 0) norm_dyn[warp * p.S_local + s] = r;
        }
        __syncwarp();
        RowFin rf{-INFINITY, 0x7fffffff, 0.0f, 0.0f, (solo && p.labels) ? p.labels[b] : -1};
        float hl = 0.0f;                                         // INFO: sum over local samples and this lane's classes of -p log p
        for (int c = lane; c < C; c += 32) {
            float mx = -INFINITY, acc = 0.0f, sp = 0.0f, sp2 = 0.0f, sl = 0.0f;
            for (int s = 0; s < p.S_local; ++s) {
                const float l = p.logits[((size_t)s * nrows + bl) * C + c];
                float pr, lp;
                if (p.normalized) { pr = softplus_f(l) / norm_dyn[warp * p.S_local + s]; lp = logf(pr); }
                else { lp = l - norm_dyn[warp * p.S_local + s]; pr = expf(lp); }            // log_softmax (main_bayesian.py:49)
                if (lp > mx) { acc = acc * expf(mx - lp) + 1.0f; mx = lp; }  // online logsumexp over the samples
                else if (lp > -INFINITY) acc += expf(lp - mx);               // lp == -inf: a probability of exactly 0 adds nothing
                sp += pr; sp2 += pr * pr; sl += l;
                if constexpr (INFO) hl -= pr > 0.0f ? pr * lp : 0.0f;       // 0 log 0 = 0, not 0 * -inf
            }
            const size_t e = (size_t)b * C + c;
            if (solo) { fin_elem(rf, e, c, mx, acc, sp, sp2, sl); continue; }
            for (int q = 0; q < p.world; ++q) {
                unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.peer[q] + MCX_CTRL_BYTES) + slot_off + (size_t)src() * rank_floats;
                st_ll(dst + e, mx, seq); st_ll(dst + BC + e, acc, seq);
                if (p.want_moments) { st_ll(dst + 2 * (size_t)BC + e, sp, seq); st_ll(dst + 3 * (size_t)BC + e, sp2, seq); st_ll(dst + 4 * (size_t)BC + e, sl, seq); }
            }
        }
        float hloc = 0.0f;                                       // INFO: sum over the local samples of H[p_hat_s]
        if constexpr (INFO) {
            hloc = warp_sum(hl);
            if (!solo && lane < p.world)                         // a rank without samples pushes 0
                st_ll(reinterpret_cast<unsigned long long*>(p.peer[lane] + MCX_CTRL_BYTES) + slot_off + (size_t)src() * rank_floats +
                          mcx_info_off(B, C, p.want_moments) + b, hloc, seq);
        }
        if (solo) fin_row(rf, b, hloc);
        __syncwarp();
    }
    float kl_solo = 0.0f;
    if (solo) {
        if (blockIdx.x == 0 && threadIdx.x == 0) for (int i = 0; p.kl && i < p.n_kl; ++i) kl_solo += __ldg(p.kl + i);
        kl_solo *= (float)p.S_local;
    } else {
        // this rank's KL contribution: S_local * kl (row blocks: the group's block-0 rank, so each group counts once)
        if (blockIdx.x == 0 && threadIdx.x < p.world && (!SHARD || p.block == 0)) {
            unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.peer[threadIdx.x] + MCX_CTRL_BYTES) + slot_off + (size_t)src() * rank_floats;
            float one = 0.0f;
            for (int i = 0; p.kl && i < p.n_kl; ++i) one += __ldg(p.kl + i);
            st_ll(dst + (size_t)mcx_planes(p.want_moments) * BC, (float)p.S_local * one, seq);
        }
        if (tracer) tr[1] = (long long)globaltimer_ns();
        // ---- (4) finish: fixed rank (row blocks: group) order => bitwise identical on every rank --------------
        for (int b = b0 + warp; b < b1; b += nwarp) {
            RowFin rf{-INFINITY, 0x7fffffff, 0.0f, 0.0f, p.labels ? p.labels[b] : -1};
            for (int c = lane; c < C; c += 32) {
                const size_t e = (size_t)b * C + c;
                // the words of this element from up to 8 ranks in flight at once (one L2 round trip), stragglers polled;
                // ranks merged in ascending order with the online logsumexp update: same operations on every rank
                float M = -INFINITY, tot = 0.0f, mom[3] = {0.0f, 0.0f, 0.0f};
                for (int q0 = 0; q0 < nsrc(); q0 += 8) {
                    unsigned long long wm[8], wa[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (q0 + j >= nsrc()) continue;
                        const unsigned long long* r = rx + (size_t)(q0 + j) * rank_floats + e;
                        wm[j] = ld_ll(r); wa[j] = ld_ll(r + BC);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (q0 + j >= nsrc()) continue;
                        const unsigned long long* r = rx + (size_t)(q0 + j) * rank_floats + e;
                        const float mq = ll_value(wm[j], r), aq = ll_value(wa[j], r + BC);
                        if (aq > 0.0f) {
                            if (mq > M) { tot = tot * expf(M - mq) + aq; M = mq; }
                            else tot += aq * expf(mq - M);
                        }
                    }
                }
                if (p.want_moments) {
#pragma unroll
                    for (int pl = 0; pl < 3; ++pl)
                        for (int q0 = 0; q0 < nsrc(); q0 += 8) {
                            unsigned long long w[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j)
                                if (q0 + j < nsrc()) w[j] = ld_ll(rx + (size_t)(q0 + j) * rank_floats + (size_t)(2 + pl) * BC + e);
#pragma unroll
                            for (int j = 0; j < 8; ++j)
                                if (q0 + j < nsrc()) mom[pl] += ll_value(w[j], rx + (size_t)(q0 + j) * rank_floats + (size_t)(2 + pl) * BC + e);
                        }
                }
                const float sp = mom[0], sp2 = mom[1], sl = mom[2];
                fin_elem(rf, e, c, M, tot, sp, sp2, sl);
            }
            float hsum = 0.0f;
            if constexpr (INFO) {       // lane q fetches rank q's word (one round trip); every lane adds them in rank order
                float hq = 0.0f;
                if (lane < nsrc()) {
                    const unsigned long long* w = rx + (size_t)lane * rank_floats + mcx_info_off(B, C, p.want_moments) + b;
                    hq = ll_value(ld_ll(w), w);
                }
                for (int q = 0; q < nsrc(); ++q) hsum += __shfl_sync(0xffffffffu, hq, q);
            }
            fin_row(rf, b, hsum);
        }
    }
    // ---- (5) cross-CTA finish (deterministic order), KL, ELBO head, sequence number ------------------------
    if (!METRICS && solo && !(p.head && p.labels)) {
        // nothing crosses CTAs: KL / Philox base by one thread; the sequence number (slot choice, handshake) is unused
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            if (p.kl_out) *p.kl_out = kl_solo * inv_S;                    // main_bayesian.py:51  (kl / num_ens)
            if (p.noise_base) *p.noise_base += p.noise_inc;
        }
        tl_exit(p.tl);
        return;
    }
    if (tracer) tr[5] = (long long)globaltimer_ns();
    const bool want_head = p.head && p.labels;
    double nll_cta = 0.0, hit_cta = 0.0;
    if (want_head) {
        nll_cta = block_sum(METRICS && lane ? 0.0 : nll_acc, red);     // the head: lane 0's only
        __syncthreads();
        hit_cta = block_sum(METRICS && lane ? 0.0 : hit_acc, red);
    } else {
        __syncthreads();                 // the last CTA's bookkeeping below must follow every thread's reads of this launch's slot
    }
    unsigned int* mcm_last = reinterpret_cast<unsigned int*>(mcm_cta + MCM_PART);
    if constexpr (METRICS) {             // this CTA's partials: its warps' in warp order (published before the CTA counts in)
        for (int w = 0; w < nwarp; ++w) {
            if (warp == w && lane < MCM_PART / 2) { mcm_cta[2 * lane] += nll_acc; mcm_cta[2 * lane + 1] += hit_acc; }
            __syncthreads();
        }
        if (threadIdx.x < MCM_PART) {
            p.metrics[MCM_SCRATCH + blockIdx.x * MCM_PART + threadIdx.x] = mcm_cta[threadIdx.x];
            __threadfence();
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // (a fence here also waits for the acknowledgements of this CTA's NVLink stores: only where something is published)
        if (want_head) { p.head_partials[2 * blockIdx.x] = nll_cta; p.head_partials[2 * blockIdx.x + 1] = hit_cta; __threadfence(); }
        const unsigned int prev = atomicAdd(p.done, 1u);
        if constexpr (METRICS) *mcm_last = prev == gridDim.x - 1;
        if (prev == gridDim.x - 1) {
            if (want_head) __threadfence();
            float klsum = 0.0f;
            if (solo) {
                for (int i = 0; p.kl && i < p.n_kl; ++i) klsum += __ldg(p.kl + i);
                klsum *= (float)p.S_local;
            } else {
                for (int q = 0; q < nsrc(); ++q) { const unsigned long long* w = rx + (size_t)q * rank_floats + (size_t)mcx_planes(p.want_moments) * BC; klsum += ll_value(ld_ll(w), w); }
            }
            const float kl = klsum * inv_S;                               // main_bayesian.py:51  (kl / num_ens)
            if (p.kl_out) *p.kl_out = kl;
            if (p.head && p.labels) {
                double nll = 0.0, hit = 0.0;
                for (unsigned int i = 0; i < gridDim.x; ++i) { nll += ((volatile double*)p.head_partials)[2 * i]; hit += ((volatile double*)p.head_partials)[2 * i + 1]; }
                const float nllf = (float)(nll / (double)B);              // F.nll_loss(..., reduction='mean')
                p.head[0] = nllf * p.train_size + p.beta * kl;            // metrics.py:14
                p.head[1] = nllf;
                p.head[2] = (float)(hit / (double)B);                     // metrics.py:23-24
                p.head[3] = p.beta * kl;
            }
            if constexpr (METRICS) {
                __threadfence();                                          // the other CTAs' partials, read below
                p.metrics[0] += 1.0; p.metrics[1] += (double)B; p.metrics[4] += (double)klsum;   // validate_model's kl: sum_j kl_j
            }
            if (p.noise_base) *p.noise_base += p.noise_inc;               // the next step's kernels draw fresh Philox streams
            *p.done = 0u;
            *p.seq = seq;
        }
    }
    if constexpr (METRICS) {             // the last CTA: every partial over the CTAs in index order, into the accumulator
        __syncthreads();
        if (*mcm_last && threadIdx.x < MCM_PART) {
            double s = 0.0;
            for (unsigned int i0 = 0; i0 < gridDim.x; i0 += 8) {      // 8 loads in flight (L2: the other CTAs' fenced stores)
                double v[8];
#pragma unroll
                for (unsigned int j = 0; j < 8; ++j)
                    v[j] = i0 + j < gridDim.x ? __ldcg(p.metrics + MCM_SCRATCH + (i0 + j) * MCM_PART + threadIdx.x) : 0.0;
#pragma unroll
                for (int j = 0; j < 8; ++j) s += v[j];
            }
            p.metrics[MCM_HEAD + threadIdx.x] += s;
            if (threadIdx.x < 2) p.metrics[2 + threadIdx.x] += s / (double)B;   // the step's nll and accuracy means (head)
        }
    }
    tl_exit(p.tl);
}

}  // namespace bbb
