// The low-latency ("LL") transport of the Monte-Carlo exchange (mc_head.cuh) and the logit gather (mc_gather.cuh).
//
// Every float travels as ONE 8-byte store {value bits, sequence number} into a peer's receive buffer (peer-mapped memory,
// CUDA IPC).  8-byte stores are single-copy atomic over NVLink, so the receiver polls each word until its tag equals the
// launch's sequence number -- no fence, no separate flag, no CTA barrier between the push and the read.  Launch k of a
// rank uses slot k & 1 of its buffer; a peer can be at most one launch ahead (it cannot finish launch k+1 before it has
// OUR launch k+1 words, which we send after we finished reading k), so the buffers are reused with no reset.
#pragma once
#include "common.cuh"

namespace bbb {

__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned int seq) {
    const unsigned long long w = ((unsigned long long)seq << 32) | (unsigned long long)__float_as_uint(v);
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_ll(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// The value of word `w` (already loaded once as `v`) once its tag says it belongs to launch `seq`.  Never hangs: a peer
// that does not deliver within timeout_ns is counted in *timeouts and the stale value returned (the launch's results are
// then invalid).
// PER_LAUNCH: the time-out bounds the launch, not each word.  `timeouts_before` is *timeouts as the launch found it; once
// any wait of the launch has given up (the counter moved), the other waits give up too, uncounted, and later words are
// taken as they are -- a thread that owns many words of a lost peer would otherwise wait timeout_ns for each of them.
template <bool PER_LAUNCH = false>
__device__ __forceinline__ float ll_wait(unsigned long long v, const unsigned long long* w, unsigned int seq,
                                         unsigned long long timeout_ns, unsigned int* timeouts,
                                         unsigned int timeouts_before = 0) {
    if ((unsigned int)(v >> 32) != seq) {
        if constexpr (PER_LAUNCH)
            if (*(volatile unsigned int*)timeouts != timeouts_before) return __uint_as_float((unsigned int)v);
        const unsigned long long t0 = globaltimer_ns();
        unsigned int spins = 0;
        while ((unsigned int)((v = ld_ll(w)) >> 32) != seq) {
            __nanosleep(64);          // the SM is shared with the next step's kernels (overlap mode): do not hammer the LSU
            if ((++spins & 63u) == 0u && globaltimer_ns() - t0 > timeout_ns) { atomicAdd(timeouts, 1u); break; }
            if constexpr (PER_LAUNCH)
                if ((spins & 63u) == 0u && *(volatile unsigned int*)timeouts != timeouts_before) break;
        }
    }
    return __uint_as_float((unsigned int)v);
}

}  // namespace bbb
