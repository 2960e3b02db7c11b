// peer_reduce.cuh - the multi-GPU exchange step of the path, inside the reducing kernel.
//
// SURVEY.md §8e: the path shards by contiguous source-point blocks and has exactly ONE exchange per ICP iteration -
// the sum over ranks of the 27 + 5 accumulators (the OpenMP `reduction(+: ...)` of icp_test_runner.cpp:1714 and
// SymmetricHessianComputer::join, hessian_computer.h:103-108).  256 B per rank: pure latency.  A separate
// ncclAllReduce kernel behind the reduction adds a launch and a collective to every iteration, so the exchange lives
// in the LAST BLOCK of the reducing kernel instead:
//
//   every rank owns an 8 KB mailbox in its own HBM, mapped into every peer's address space (cudaIpc handles
//   exchanged once in dcreg_comm_init; NVLink / NVSwitch P2P stores);
//   epoch e (same on all ranks: every rank runs the same sequence of reductions):
//     post : warp q of the last block stores this rank's 32 packed totals into rank q's mailbox slot
//            pkt[e & 1][my_rank][0..63] as 64 self-validating 8-byte packets {32 data bits, epoch}: an aligned 8-byte
//            store is single-copy atomic, so a packet is either old or complete - no fence, no separate flag, one
//            NVLink store latency (the "LL" idea of collective libraries);
//     wait : warp q spins on ITS OWN mailbox's pkt[e & 1][q][2 lane], [2 lane + 1] until both carry epoch e and
//            reassembles the double;
//     sum  : in rank order 0..N-1 - the same order on every rank, so all ranks hold bit-identical sums and the
//            solve that follows (K2, redundantly on every rank) yields bit-identical poses: no broadcast needed.
//   Two slots (epoch parity) suffice: a rank can only post epoch e + 1 after it has received every peer's epoch e,
//   and a peer posts epoch e only after it finished reading epoch e - 1 (tests/test_peer_protocol.py runs a model of
//   this under adversarial interleavings).
// No rank waits before it has posted, so the exchange cannot deadlock; a peer that never posts (crashed process)
// trips a 4 s globaltimer timeout, which raises `error` in the mailbox instead of hanging the GPU.
// NCCL (dcreg_b200.cu: nccl_allreduce_acc) remains as the fallback when peer mapping is unavailable.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace peer {

constexpr int kMaxRanks = 8;     // one warp of the 256-thread last block per rank
constexpr int kVals = 32;        // k1s::kPk packed totals

struct Mailbox {
    unsigned long long pkt[2][kMaxRanks][2 * kVals];   // written by peer r: {low / high half of a double, epoch} packets
    unsigned int epoch;                  // this rank's own epoch counter (local)
    unsigned int error;                  // != 0: a wait timed out
    unsigned int pad[6];
};

struct View {
    int nranks;                          // <= 1: no exchange
    int rank;
    Mailbox* box[kMaxRanks];             // box[r]: rank r's mailbox in THIS process's address space (box[rank] is local)
};

__device__ __forceinline__ void st_relaxed_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// This rank's epoch counter, to be read at KERNEL START by every thread that may end up in the last block (one L2 load,
// long finished when the exchange needs it: not a round trip on the critical path).
__device__ __forceinline__ unsigned int load_epoch(const View& pv) {
    return pv.nranks > 1 ? pv.box[pv.rank]->epoch : 0u;
}

// All 256 threads of the (single) last block call this.  fin[32] (shared memory): in = this rank's packed totals,
// out = the sum over ranks in rank order.  red: shared scratch [kMaxRanks][32].  epoch_in = load_epoch() of this launch.
__device__ __forceinline__ void all_reduce32(const View& pv, double* fin, double (*red)[kVals], unsigned int epoch_in) {
    if (pv.nranks <= 1) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = (int)(blockDim.x >> 5);
    Mailbox* mine = pv.box[pv.rank];
    const unsigned int e = epoch_in + 1u;
    const double v = fin[lane];
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    const unsigned long long tag = (unsigned long long)e << 32;
    for (int q = warp; q < pv.nranks; q += nwarps) {    // post
        if (q == pv.rank) { red[q][lane] = v; continue; }
        unsigned long long* dst = pv.box[q]->pkt[e & 1u][pv.rank];
        st_relaxed_sys(dst + 2 * lane, (bits & 0xffffffffull) | tag);
        st_relaxed_sys(dst + 2 * lane + 1, (bits >> 32) | tag);
    }
    for (int q = warp; q < pv.nranks; q += nwarps) {    // wait
        if (q == pv.rank) continue;
        const unsigned long long* src = mine->pkt[e & 1u][q];
        unsigned long long p0, p1, t0 = 0;
        while (true) {
            p0 = ld_relaxed_sys(src + 2 * lane);
            p1 = ld_relaxed_sys(src + 2 * lane + 1);
            if ((unsigned int)(p0 >> 32) == e && (unsigned int)(p1 >> 32) == e) break;
            unsigned long long now;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000ull) { mine->error = 1u + (unsigned)q; p0 = p1 = 0; break; }
        }
        red[q][lane] = __longlong_as_double((long long)((p0 & 0xffffffffull) | (p1 << 32)));
    }
    __syncthreads();
    if (tid < kVals) {
        double s = 0.0;
        for (int r = 0; r < pv.nranks; ++r) s += red[r][tid];
        fin[tid] = s;
    }
    if (tid == 0) mine->epoch = e;
    __syncthreads();
}

}  // namespace peer
