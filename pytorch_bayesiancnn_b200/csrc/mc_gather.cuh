// Gather of a sharded Monte-Carlo step's per-sample logits onto every rank (bbb_mc_logit_gather), for the sample banks
// (ProbBank, LogitBank) that need all S samples of every image.
//
// World = Rs sample groups x Rb row blocks, as the exchange (mc_head.cuh, SHARD): rank r is sample group g = r % Rs
// (global samples g, g + Rs, ..) and row block k = r / Rs (images [row0, row0 + rows)).  Its logits are
// [S_local, rows, C]; local element (i, b, c) is global element (g + i Rs, row0 + b, c) of [S, B, C].
//
// Receive buffer of one rank: u64 data[2 slots][S * B * C], one LL word (ll.cuh) per float at its GLOBAL position, so
// every word has exactly one sender.  (1) every CTA pushes its share of the local elements into every rank's buffer
// (st.relaxed.sys, no fence, no flag); (2) it then polls its share of the S * B * C words of its own buffer until each
// carries this launch's sequence number and writes the plain fp32 value, bits unchanged (NaN, inf, -0.0 included);
// (3) the last CTA to finish advances the sequence number.  A CTA pushes all of its share before it polls, and the
// grid is co-resident, so every word a CTA waits for is stored by a CTA that runs.
#pragma once
#include "common.cuh"
#include "fwd_tc.cuh"      // pdl_wait
#include "ll.cuh"
#include "mc_head.cuh"     // MCX_MAX_RANKS

namespace bbb {

// At most MCG_MAX_CTAS CTAs of MCG_THREADS, <= 64 registers and a few bytes of static shared memory: four fit on an SM,
// so even 16 ranks' grids (512 CTAs) are co-resident on one 132-SM device and a CTA spinning on a peer's word never
// keeps that peer's producer off an SM.
constexpr int MCG_THREADS = 256, MCG_MAX_CTAS = 32, MCG_BATCH = 8;

__host__ __device__ inline size_t mcg_words(int S, int B, int C) { return (size_t)S * (size_t)B * (size_t)C; }

struct McgArgs {
    const float* logits;            // [S_local, rows, C] this rank's samples and rows; nullable when S_local == 0
    int S_local, S, B, C;
    int groups, group, row0, rows;  // Rs, g, and this rank's row block
    int rank, world;
    unsigned char* peer[MCX_MAX_RANKS];   // receive buffers; peer[rank] is the local one
    unsigned int* seq;              // local device counter: launches completed so far
    unsigned int* done;             // local device counter (zeroed once): CTAs finished in this launch
    unsigned int* timeouts;         // local device counter: waits that gave up (the output is then invalid)
    unsigned int* timeouts_before;  // local device word: *timeouts when this launch began (written by the last launch)
    unsigned long long timeout_ns;
    float* out;                     // [S, B, C]
};

__global__ void __launch_bounds__(MCG_THREADS, 4)
mc_logit_gather_kernel(const McgArgs a) {
    __shared__ unsigned int seq_sh, before_sh;
    pdl_wait();                     // launched with programmatic serialization: the logits come from the predecessor
    if (threadIdx.x == 0) { seq_sh = *a.seq + 1u; before_sh = *a.timeouts_before; }
    __syncthreads();
    const unsigned int seq = seq_sh, before = before_sh;
    const size_t total = mcg_words(a.S, a.B, a.C);
    const size_t slot = (size_t)(seq & 1u) * total;
    const size_t tid = (size_t)blockIdx.x * MCG_THREADS + threadIdx.x, stride = (size_t)gridDim.x * MCG_THREADS;

    // (1) push: local sample i's rows are contiguous in [S, B, C] at (g + i Rs, row0); every peer, starting with the next
    // rank, so that the ranks do not all store to the same peer first
    const size_t rowc = (size_t)a.rows * a.C;
    for (int i = 0; i < a.S_local; ++i) {
        const float* src = a.logits + (size_t)i * rowc;
        const size_t dst0 = slot + ((size_t)(a.group + i * a.groups) * a.B + a.row0) * a.C;
        for (size_t e0 = tid; e0 < rowc; e0 += MCG_BATCH * stride) {
            float v[MCG_BATCH];
#pragma unroll
            for (int j = 0; j < MCG_BATCH; ++j) {
                const size_t e = e0 + j * stride;
                v[j] = e < rowc ? __ldg(src + e) : 0.0f;
            }
            int q = a.rank;
            for (int k = 0; k < a.world; ++k) {
                q = q + 1 == a.world ? 0 : q + 1;
                unsigned long long* d = reinterpret_cast<unsigned long long*>(a.peer[q]) + dst0;
#pragma unroll
                for (int j = 0; j < MCG_BATCH; ++j) {
                    const size_t e = e0 + j * stride;
                    if (e < rowc) st_ll(d + e, v[j], seq);
                }
            }
        }
    }
    // (2) read: MCG_BATCH words in flight per thread (one round trip), stragglers polled; a lost peer costs the launch one
    // time-out, not one per word (ll_wait<PER_LAUNCH>)
    const unsigned long long* rx = reinterpret_cast<const unsigned long long*>(a.peer[a.rank]) + slot;
    for (size_t e0 = tid; e0 < total; e0 += MCG_BATCH * stride) {
        unsigned long long w[MCG_BATCH];
#pragma unroll
        for (int j = 0; j < MCG_BATCH; ++j) {
            const size_t e = e0 + j * stride;
            if (e < total) w[j] = ld_ll(rx + e);
        }
#pragma unroll
        for (int j = 0; j < MCG_BATCH; ++j) {
            const size_t e = e0 + j * stride;
            if (e < total) a.out[e] = ll_wait<true>(w[j], rx + e, seq, a.timeout_ns, a.timeouts, before);
        }
    }
    // (3) the last CTA: this launch is done on this rank (the next launch reads the sequence number and the time-out
    // count it starts from in stream order)
    __syncthreads();
    if (threadIdx.x == 0) __threadfence();      // this CTA's time-outs are counted before it counts in
    if (threadIdx.x == 0 && atomicAdd(a.done, 1u) == gridDim.x - 1) {
        __threadfence();
        *a.done = 0u;
        *a.timeouts_before = *(volatile unsigned int*)a.timeouts;
        *a.seq = seq;
    }
}

}  // namespace bbb
