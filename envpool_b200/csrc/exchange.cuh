// Peer exchange: the one data-path collective of the sharded step (SURVEY.md 8(e)).
//
// The reference has no counterpart (it is single-process); north_star asks that after every
// step each GPU holds the outputs of ALL envs.  Every rank owns one "gather" allocation
//
//     slot[D][world][slice_bytes] | data_flag[D][16] | ack_flag[16] | ctl | PeerView[D]
//
// mapped into every peer (CUDA IPC between processes, plain pointers inside one process).
// slice = the packed output slab (all 13 columns at their slab offsets) + one extra "wire"
// column `packed[N]` (int32: elapsed_step << 2 | trunc << 1 | done).
//
// What crosses NVLink per env-step is only what a peer cannot know: the env keys (obs and
// info columns), `reward` and the packed word -- CartPole 24 B instead of the slab's 42 B.
// info:env_id / info:players.env_id are constants (written into every slot once, at attach
// time); elapsed_step, done, trunc, discount and step_type are re-expanded from the packed
// word on the receiving GPU (`wait_derive_kernel`), where the bytes cost local HBM, not link.
//
// A step writes its slab straight into slot[t % D][rank] of the LOCAL allocation (no staging
// copy) and the wire columns go into slot[t % D][rank] of every peer with 16-byte stores,
// after which the step's sequence number is published in data_flag[rank] of every rank.
// The one producer of the peer stores is `push_kernel` (capi.cu), a copy kernel of its own
// behind the step kernel: on the step's stream for direct steps and uncaptured chains, on
// branches beside the step chain in captured chains (capi.cu `run_chain`).  The step kernels
// know nothing of the exchange beyond the packed wire column they write.
// Flow control.  D slots form a ring, so a rank may run up to D-1 steps ahead of the slowest
// consumer: step t+1 computes and pushes while the data of step t is still in flight or being
// consumed (the sender never waits for the transfer of the previous step).  Slot t % D may be
// overwritten by step t + D only after every rank has released step t; a rank releases by
// publishing ack_flag (its wait kernel for step u first stores "steps < u are consumed" into
// ack_flag[rank] of every rank).  The pushing CTAs check the credit (`peer_credit`: every
// ack >= t - D + 1) right before their first peer store -- a local L2 read that is almost
// always true at once; with step/wait strictly alternating on one stream it always is.
//
// Why not ncclAllGather: its per-call protocol latency for the CartPole slab is many times the
// step itself; the peer stores cost the NVLink time of the payload and one flag round trip.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace epb {

constexpr int kMaxPeers = 16;
constexpr int kMaxDepth = 8;

constexpr int kMaxCols = 13;  // wire columns: reward, the env keys (Go: 10), the packed word

struct ExchangeCtl {
  unsigned int blocks_done[kMaxDepth];       // last-block-done counter of the push into slot s
  unsigned int wait_blocks;                  // ... and of the wait kernel
  unsigned int pad0;
  // step index the NEXT push into ring slot s carries (s, s + D, s + 2D, ...): pushes into
  // different slots may be in flight together (captured chains run them on several branches),
  // so the step a pushing kernel works on cannot be a single running counter
  unsigned long long slot_step[kMaxDepth];
  unsigned long long seq;      // steps published by this rank (highest step + 1)
  unsigned long long waited;   // steps whose wait kernel has finished on this rank
  int error;                   // 1 = a wait timed out
  int pad2;
  // optional timeline (ENVPOOL_B200_EXCHANGE_TRACE=1; profiles/exchange_trace.py): 8 globaltimer
  // stamps per exchanged step: [0] push kernel starts, [1] its credit is there, [2] its last
  // CTA publishes, [3] wait kernel starts, [4] last peer flag seen, [5] wait kernel ends,
  // [6] CTA 0 of the push has issued its stores, [7] CTA 0 is past its system fence
  long long* trace;
  long long trace_steps;
};
__device__ __forceinline__ long long exchange_now() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void exchange_stamp(ExchangeCtl* ctl, unsigned long long step, int k,
                                               bool take_max = false) {
  if (ctl->trace && (long long)step < ctl->trace_steps) {
    long long* p = ctl->trace + step * 8 + k;
    if (take_max) atomicMax(p, exchange_now());
    else *p = exchange_now();
  }
}

struct PeerView {
  char* slice[kMaxPeers];                // slot[s][rank] in the allocation of rank g
  unsigned long long* flag[kMaxPeers];   // &data_flag[rank] in the allocation of rank g
  ExchangeCtl* ctl;                      // this rank's control block
  const unsigned long long* ack;         // this rank's ack_flag[world] (peers write it)
  long long timeout_ns;                  // bound of the credit wait
  int world;
  int rank;
  int depth;                             // ring slots
  int slot;                              // the ring slot this view describes
  // wire columns (forwarded to peers): byte offset in the slice and bytes per row
  int ncols;
  int col_rb[kMaxCols];
  int64_t col_off[kMaxCols];
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void st_relaxed_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// elapsed_step << 2 | trunc << 1 | done: everything the common columns are made of
__device__ __forceinline__ int32_t pack_wire(int cur, int done, int trunc) {
  return (cur << 2) | (trunc << 1) | done;
}

// Credit of step t (t = ctl->slot_step[slot], the step this push into the slot carries): slot t % D may be
// overwritten on rank g once g has released step t - D, i.e. ack_flag[g] >= t - D + 1.  The
// flags live in THIS rank's memory (peers store into them), so the poll is a local L2 read
// and, with any slack in the ring, true on the first look.  Lanes 0..world-1 of the CTA poll;
// bounded like every wait of the exchange.  slot_step[slot] cannot change while a CTA is here:
// it is bumped by the last CTA of this push to finish, and this one has not finished.  Deadlock-free: the
// releases a rank waits for are published by kernels of OTHER GPUs, and its own release of
// step t - D precedes this kernel in stream / graph order.
__device__ __forceinline__ void peer_credit(const PeerView* __restrict__ pv) {
  const int tid = threadIdx.x;
  if (tid < pv->world) {  // own release included: the local consumer may sit on another stream
    const unsigned long long t = pv->ctl->slot_step[pv->slot];
    if (t >= (unsigned long long)pv->depth) {
      const unsigned long long need = t - pv->depth + 1;
      long long t0 = 0;
      bool timing = false;
      while (ld_acquire_sys(pv->ack + tid) < need) {
        long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (!timing) {
          t0 = t1;
          timing = true;
        } else if (t1 - t0 > pv->timeout_ns) {
          atomicExch(&pv->ctl->error, 1);
          break;
        }
        __nanosleep(32);
      }
    }
  }
}

// Last-block-done publication.  Per CTA: barrier (every peer store of the CTA is issued before
// it), then ONE thread fences at system scope and counts the CTA -- a fence is cumulative: it
// orders every write that happens-before it, and the barrier puts the whole CTA's stores there
// (the release pattern of cooperative-groups grid sync and of CUTLASS's semaphore, at .sys
// scope).  The first version had EVERY thread fence: 2048 warps issuing MEMBAR.SYS behind
// in-flight NVLink stores was the dominant cost of a small exchange.  The CTA that completes the count bumps the sequence number,
// fences once more (acquire side of the ticket, release side of the flags) and raises
// data_flag[slot][rank] = step + 1 on every rank with relaxed stores (a release per flag would pay one NVLink
// round trip per peer).  Call with all threads of the CTA.
__device__ __forceinline__ void peer_publish(const PeerView* __restrict__ pv) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    ExchangeCtl* ctl = pv->ctl;
    const int slot = pv->slot;
    if (blockIdx.x == 0) exchange_stamp(ctl, ctl->slot_step[slot], 7);
    unsigned int ticket = atomicAdd(&ctl->blocks_done[slot], 1u);
    if (ticket == gridDim.x - 1) {
      ctl->blocks_done[slot] = 0;
      const unsigned long long t = ctl->slot_step[slot];
      exchange_stamp(ctl, t, 2);
      ctl->slot_step[slot] = t + pv->depth;
      atomicMax(&ctl->seq, t + 1);
      __threadfence_system();
      const int world = pv->world;
      for (int g = 0; g < world; ++g) st_relaxed_sys(pv->flag[g], t + 1);
    }
  }
}

}  // namespace epb
