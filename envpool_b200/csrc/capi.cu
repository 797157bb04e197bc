// envpool_b200 C ABI (include/envpool_b200.h): pool lifetime, key tables, the host-buffer
// send/recv path (pinned staging + one packed D2H per batch) and the device-resident
// step / rollout path.  This file is the GPU-side replacement for the reference's
// AsyncEnvPool + ActionBufferQueue + StateBufferQueue (envpool/core/async_envpool.h,
// action_buffer_queue.h, state_buffer_queue.h): the "queue" is a CUDA stream, the
// "state buffer" is a packed output slab in HBM mirrored into recycled pinned host slabs.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/envpool_b200.h"
#include "common.cuh"
#include "mujoco.cuh"

namespace epb {

__global__ void seed_kernel(StateView sv, int base_seed, const int32_t* env_seed) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= sv.n_envs) return;
  // Env::ResolveSeed (core/env.h:101-111): env_seed[env_id] or seed + env_id
  uint32_t s = env_seed ? (uint32_t)env_seed[e] : (uint32_t)(base_seed + sv.env_id_offset + e);
  // chunked layout (common.cuh): chunk c of env e is the 8 words at ((c*N + e)*8)
  const int64_t N = sv.n_envs;
  uint32_t w[8];
  for (int c = 0; c < kMtN / 8; ++c) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = c * 8 + k;
      if (i > 0) s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)i;
      w[k] = s;
    }
    uint4* dst = reinterpret_cast<uint4*>(sv.mt + ((int64_t)c * N + e) * 8);
    dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
    dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
  }
  sv.mt_idx[e] = 0;  // std::mt19937 starts exhausted: the first draw regenerates word 0
  sv.flags[e] = -1;  // current_step_ = -1 (env.h:81), done_ = true (cartpole.h:67)
}

thread_local std::string g_err;

static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define EPB_CUDA(expr)                                                            \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess)                                                        \
      return fail(EPB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// Every entry point runs on the pool's device but leaves the caller's current device as it
// found it (a host process may drive several pools / use torch on another GPU).
struct DeviceGuard {
  int prev = -1;
  cudaError_t status;
  explicit DeviceGuard(int dev) {
    status = cudaGetDevice(&prev);
    if (status == cudaSuccess && prev != dev) status = cudaSetDevice(dev);
    else if (status == cudaSuccess) prev = -1;  // nothing to restore
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

struct Key {
  const char* name;
  int dtype, ndim, shape[3], row_bytes;
  int64_t off;
  int players;  // rows per env row: KindDesc::players for a per-player column, else 1
};

static int dtype_size(int d) { return d == EPB_F64 ? 8 : d == EPB_BOOL ? 1 : 4; }

// What a cached chain graph was captured for.
struct ChainKey {
  const void* actions;
  int T, t0, K, mark0, mark1, exchange, phase;
  cudaStream_t stream;
  bool operator==(const ChainKey& o) const {
    return actions == o.actions && T == o.T && t0 == o.t0 && K == o.K && mark0 == o.mark0 &&
           mark1 == o.mark1 && exchange == o.exchange && phase == o.phase && stream == o.stream;
  }
};

struct Pending {
  void* slab;
  int n;       // rows written by this send/reset
  int row0;    // rows already handed out (async mode hands out batch_size rows at a time)
  cudaEvent_t ev;
  bool ready;  // event already waited for
};

}  // namespace epb

using namespace epb;

struct epb_pool {
  int kind = 0;
  epb_config cfg{};
  int N = 0;
  int precision = 0;
  std::vector<Key> keys;
  Key act{};
  int64_t slab_bytes = 0;
  int NR = 0, NI = 0, real_size = 8;
  StateView sv{};
  // device allocations
  void* d_state_blob = nullptr;  // flags | mt_idx | istate | rstate | mt | (records)
  int64_t state_bytes = 0;
  char* d_slab = nullptr;
  char* d_last = nullptr;  // slab the most recent *_device launch wrote (d_slab or a gather slice)
  void* d_action = nullptr;
  int32_t* d_ids = nullptr;
  // pinned host staging
  void* h_action[2] = {nullptr, nullptr};
  int32_t* h_ids[2] = {nullptr, nullptr};
  cudaEvent_t h_stage_ev[2] = {nullptr, nullptr};
  int stage_flip = 0;
  std::vector<int32_t> arange;  // 0..N-1, for the identity-ids fast path
  int batch = 0;                // rows per recv; < N = async mode (async_envpool.h:93-97)
  std::vector<std::pair<void*, int>> leases;  // slab -> outstanding recv leases + queue refs
  std::vector<void*> free_slabs;
  std::vector<void*> all_slabs;
  // pinned slabs whose two id columns hold arange + env_id_offset (the full sync batch with
  // identity ids never changes them, so its D2H copy skips them)
  std::vector<void*> ids_ok_slabs;
  std::deque<Pending> pending;
  std::vector<cudaEvent_t> free_events;
  std::mutex mu;
  cudaStream_t stream = nullptr;
  KindLaunch fn{};              // the kind's kernels (common.cuh KindDesc)
  std::vector<char> params;     // family parameters (KindDesc::setup)
  // reset-ahead records (common.cuh StateView::rec, fn.refill): the refill schedule and the side
  // stream + events that put refill(t) on a parallel branch of the engine's captured step chains
  int refill_every = 8;    // a refill launch after every this many step launches (< rec_q)
  int since_refill = 0;    // step launches since the last refill
  cudaStream_t side = nullptr;
  cudaEvent_t ev_step[2] = {nullptr, nullptr}, ev_refill[2] = {nullptr, nullptr};
  // cached CUDA graphs of K-step chains (epb_step_many_device), most recent first
  struct GraphEntry {
    cudaGraphExec_t exec;
    ChainKey key;
    int64_t launches;  // kernels one replay launches
  };
  std::vector<GraphEntry> graphs;
  // timing marks inside a chain (epb_step_many_timed): timed events + the branch they are
  // recorded on
  cudaStream_t mark_side = nullptr;
  cudaEvent_t ev_mark = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  int64_t launches = 0;
  int bytes_per_step = 0;
  bool started = false;  // a step, reset or rollout has been launched
  bool imported = false;  // epb_state_import has loaded a blob (Go: with its configuration)
  // peer exchange (exchange.cuh):
  //   slot[D][world][x_slice] | data_flag[16] | ack_flag[16] | ctl | PeerView[D]
  char* x_base = nullptr;
  int x_world = 0, x_rank = 0, x_depth = 4;
  int64_t x_slice = 0;     // slab_bytes + the packed wire column
  int64_t x_data_off = 0, x_ack_off = 0, x_ctl_off = 0, x_view_off = 0, x_bytes = 0;
  char* x_peer[kMaxPeers] = {};
  bool x_ipc[kMaxPeers] = {};
  bool x_attached = false;
  long long x_timeout_ns = 10000000000LL;
  long long* x_trace = nullptr;  // ENVPOOL_B200_EXCHANGE_TRACE: device timeline, 8 stamps / step
  int64_t x_trace_steps = 0;
  uint64_t x_steps = 0;   // host count of exchanged steps; step t uses slot t % D
  uint64_t x_waited = 0;  // host count of enqueued waits
  cudaStream_t x_side = nullptr;            // wait branch of the engine-captured chains
  cudaStream_t x_push[3] = {};              // push branches of captured chains: push(k) on k % 3
  cudaEvent_t x_ev_step[kMaxDepth] = {}, x_ev_wait[kMaxDepth] = {}, x_ev_push[kMaxDepth] = {};

  int64_t x_mine(int slot) const { return ((int64_t)slot * x_world + x_rank) * x_slice; }
  ExchangeCtl* x_ctl() const { return reinterpret_cast<ExchangeCtl*>(x_base + x_ctl_off); }
  PeerView* x_view(int slot) const {
    return reinterpret_cast<PeerView*>(x_base + x_view_off) + slot;
  }

  OutView slab_view(char* base) const {
    OutView ov{};
    auto col = [&](int k) { return static_cast<void*>(base + keys[k].off); };
    ov.env_id = static_cast<int32_t*>(col(0));
    ov.players_id = static_cast<int32_t*>(col(1));
    ov.elapsed = static_cast<int32_t*>(col(2));
    ov.done = static_cast<uint8_t*>(col(3));
    ov.reward = static_cast<float*>(col(4));
    ov.discount = static_cast<float*>(col(5));
    ov.step_type = static_cast<int32_t*>(col(6));
    ov.trunc = static_cast<uint8_t*>(col(7));
    for (size_t k = 8; k < keys.size() && k < 13; ++k) ov.env[k - 8] = col((int)k);
    ov.t_stride_rows = N;
    return ov;
  }
  // env keys 5..9 of the slab at `base` (LaunchArgs::env_hi)
  void slab_hi(char* base, void* (&hi)[kEnvKeys - 5]) const {
    for (size_t k = 13; k < keys.size(); ++k) hi[k - 13] = base + keys[k].off;
  }
};

namespace {

// A per-player column of a kind with P > 1 players: its row for env row i holds the rows of
// players 0..P-1 of that env, next to each other.  `shape` is one player's row (obs already
// fills the three dims epb_key_info has); row_bytes covers all P.
Key make_key(const EnvKey& e, int players) {
  Key k{};
  k.name = e.name;
  k.dtype = e.dtype;
  k.players = e.per_player ? players : 1;
  k.ndim = e.ndim;
  k.row_bytes = dtype_size(e.dtype) * k.players;
  for (int i = 0; i < e.ndim; ++i) {
    k.shape[i] = e.shape[i];
    k.row_bytes *= e.shape[i];
  }
  return k;
}

// common_state_spec, envpool/core/env_spec.h:37-43 (leading -1 there = per player)
constexpr EnvKey kCommonKeys[] = {
    {"info:env_id", EPB_I32},           {"info:players.env_id", EPB_I32, 0, {}, true},
    {"elapsed_step", EPB_I32},          {"done", EPB_BOOL},
    {"reward", EPB_F32, 0, {}, true},   {"discount", EPB_F32, 0, {}, true},
    {"step_type", EPB_I32},             {"trunc", EPB_BOOL},
};

void build_keys(epb_pool* p, const KindDesc& d) {
  for (const EnvKey& k : kCommonKeys) p->keys.push_back(make_key(k, d.players));
  for (const EnvKey& k : d.keys)
    if (k.name) p->keys.push_back(make_key(k, d.players));
  p->act = make_key(d.action, 1);  // one action row per env row
  int64_t off = 0;
  for (Key& k : p->keys) {
    k.off = off;
    off += ((int64_t)k.row_bytes * p->N + 255) / 256 * 256;
  }
  p->slab_bytes = off;
}

void fill_id_columns(epb_pool* p, void* slab) {
  int32_t* a = reinterpret_cast<int32_t*>(static_cast<char*>(slab) + p->keys[0].off);
  int32_t* b = reinterpret_cast<int32_t*>(static_cast<char*>(slab) + p->keys[1].off);
  const int off = p->cfg.env_id_offset, P = p->keys[1].players;
  for (int i = 0; i < p->N; ++i) {
    a[i] = off + i;
    for (int j = 0; j < P; ++j) b[(int64_t)i * P + j] = off + i;
  }
}

int alloc_slab(epb_pool* p, void** out) {
  void* h = nullptr;
  cudaError_t e = cudaHostAlloc(&h, (size_t)p->slab_bytes, cudaHostAllocDefault);
  if (e != cudaSuccess)
    return fail(EPB_ERR_CUDA, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  fill_id_columns(p, h);
  p->all_slabs.push_back(h);
  p->ids_ok_slabs.push_back(h);
  *out = h;
  return EPB_OK;
}

// A free pinned slab (recycled; a new one costs milliseconds of cudaHostAlloc, which is why
// epb_create allocates the first few).  *ids_ok: its id columns already hold the identity.
int get_slab(epb_pool* p, void** out, bool* ids_ok) {
  std::lock_guard<std::mutex> lk(p->mu);
  if (!p->free_slabs.empty()) {
    *out = p->free_slabs.back();
    p->free_slabs.pop_back();
  } else {
    int rc = alloc_slab(p, out);
    if (rc != EPB_OK) return rc;
  }
  *ids_ok = false;
  for (void* s : p->ids_ok_slabs)
    if (s == *out) *ids_ok = true;
  return EPB_OK;
}
void set_ids_ok(epb_pool* p, void* slab, bool ok) {
  std::lock_guard<std::mutex> lk(p->mu);
  for (size_t i = 0; i < p->ids_ok_slabs.size(); ++i)
    if (p->ids_ok_slabs[i] == slab) {
      if (ok) return;
      p->ids_ok_slabs.erase(p->ids_ok_slabs.begin() + i);
      return;
    }
  if (ok) p->ids_ok_slabs.push_back(slab);
}

int get_event(epb_pool* p, cudaEvent_t* ev) {
  std::lock_guard<std::mutex> lk(p->mu);
  if (!p->free_events.empty()) {
    *ev = p->free_events.back();
    p->free_events.pop_back();
    return EPB_OK;
  }
  EPB_CUDA(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
  return EPB_OK;
}

// Copy the wire columns of the local slice to every peer, then publish: behind the step on its
// own stream for direct steps and uncaptured chains, and on the push branches of captured
// chains.  Column k is ceil(n * row_bytes / 16) 16-byte units (the 256-byte
// column padding absorbs the tail).
__global__ void __launch_bounds__(256)
push_kernel(const PeerView* __restrict__ pv, int n) {
  const int world = pv->world, rank = pv->rank;
  const char* __restrict__ src = pv->slice[rank];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if (blockIdx.x == 0 && threadIdx.x == 0)
    exchange_stamp(pv->ctl, pv->ctl->slot_step[pv->slot], 0);
  peer_credit(pv);
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0)
    exchange_stamp(pv->ctl, pv->ctl->slot_step[pv->slot], 1);
  for (int k = 0; k < pv->ncols; ++k) {
    const int64_t off = pv->col_off[k];
    const int64_t n16 = ((int64_t)n * pv->col_rb[k] + 15) >> 4;
    // up to four 16-byte units per thread and pass: the loads (L2 hits) first, then the stores
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n16; i0 += 4 * stride) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t i = i0 + j * stride;
        if (i < n16) v[j] = reinterpret_cast<const uint4*>(src + off)[i];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t i = i0 + j * stride;
        if (i < n16) {
#pragma unroll 1
          for (int g = 0; g < world; ++g)
            if (g != rank) reinterpret_cast<uint4*>(pv->slice[g] + off)[i] = v[j];
        }
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    exchange_stamp(pv->ctl, pv->ctl->slot_step[pv->slot], 6);
  peer_publish(pv);
}

struct WaitArgs {
  const unsigned long long* data_flag;      // [depth][kMaxPeers] in this rank's allocation
  unsigned long long* ack_dst[kMaxPeers];   // &ack_flag[rank] in the allocation of rank g
  char* slots;                              // this rank's slot[0][0]
  int64_t slice, wire_off;
  int64_t off_elapsed, off_done, off_discount, off_step_type, off_trunc;
  ExchangeCtl* ctl;
  long long timeout_ns;
  int world, rank, depth, n;
};

// Wait for step u = ctl->waited of every rank and finish its batch.  Grid (x, world):
// row g of the grid handles the slice of rank g.  First the release of everything older
// (ack = u: "steps < u are consumed here" -- the consumer of step u-1 precedes this kernel in
// stream order), then thread 0 of each CTA acquires data_flag[g] >= u + 1 (bounded: a dead
// peer sets ctl->error instead of hanging the GPU) and the CTAs of row g re-expand the common
// columns of rank g's slice from its packed wire column.  Bounded by local HBM, not the link.
template <int P>
__device__ __forceinline__ void wait_derive(const WaitArgs& a) {
  ExchangeCtl* ctl = a.ctl;
  const unsigned long long u = ctl->waited;
  const int g = blockIdx.y;
  if (blockIdx.x == 0 && g == 0 && threadIdx.x == 0) exchange_stamp(ctl, u, 3);
  if (blockIdx.x == 0 && g == 0 && (int)threadIdx.x < a.world)
    st_release_sys(a.ack_dst[threadIdx.x], u);
  if (g != a.rank) {
    if (threadIdx.x == 0) {
      long long t0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      const unsigned long long* flag = a.data_flag + (u % a.depth) * kMaxPeers + g;
      while (ld_acquire_sys(flag) < u + 1) {
        long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > a.timeout_ns) {
          atomicExch(&ctl->error, 1);
          break;
        }
        __nanosleep(32);
      }
      if (blockIdx.x == 0) exchange_stamp(ctl, u, 4, true);
    }
    __syncthreads();
    char* sl = a.slots + ((int64_t)(u % a.depth) * a.world + g) * a.slice;
    const int4* __restrict__ wire = reinterpret_cast<const int4*>(sl + a.wire_off);
    int4* elapsed = reinterpret_cast<int4*>(sl + a.off_elapsed);
    uchar4* done = reinterpret_cast<uchar4*>(sl + a.off_done);
    float4* discount = reinterpret_cast<float4*>(sl + a.off_discount);  // P float4 per quad
    int4* step_type = reinterpret_cast<int4*>(sl + a.off_step_type);
    uchar4* trunc = reinterpret_cast<uchar4*>(sl + a.off_trunc);
    const int n4 = (a.n + 3) >> 2;  // the tail quad stays inside the 256-byte column padding
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
      const int4 w = __ldcg(wire + i);
      const int ww[4] = {w.x, w.y, w.z, w.w};
      int el[4], st[4];
      unsigned char dn[4], tr[4];
      float dc[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        dn[j] = (unsigned char)(ww[j] & 1);
        tr[j] = (unsigned char)((ww[j] >> 1) & 1);
        el[j] = ww[j] >> 2;
        dc[j] = dn[j] ? 0.0f : 1.0f;
        st[j] = el[j] == 0 ? 0 : (dn[j] ? 2 : 1);
      }
      elapsed[i] = make_int4(el[0], el[1], el[2], el[3]);
      done[i] = make_uchar4(dn[0], dn[1], dn[2], dn[3]);
      if constexpr (P == 1) {
        discount[i] = make_float4(dc[0], dc[1], dc[2], dc[3]);
      } else {  // write_common_pair: player 1's discount is 0
        discount[2 * i] = make_float4(dc[0], 0.0f, dc[1], 0.0f);
        discount[2 * i + 1] = make_float4(dc[2], 0.0f, dc[3], 0.0f);
      }
      step_type[i] = make_int4(st[0], st[1], st[2], st[3]);
      trunc[i] = make_uchar4(tr[0], tr[1], tr[2], tr[3]);
    }
  }
  // last block done: the next wait kernel handles step u + 1
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    if (atomicAdd(&ctl->wait_blocks, 1u) == total - 1) {
      exchange_stamp(ctl, u, 5);
      ctl->wait_blocks = 0;
      ctl->waited = u + 1;
    }
  }
}
__global__ void __launch_bounds__(256) wait_derive_kernel(WaitArgs a) { wait_derive<1>(a); }
// two players per env: the discount column holds two rows per env (write_common_pair)
__global__ void __launch_bounds__(256) wait_derive_pair_kernel(WaitArgs a) { wait_derive<2>(a); }

// info:env_id / info:players.env_id of every rank's slice in every slot never change:
// rank g owns the global ids [id0 + g * n, id0 + (g + 1) * n).
// info:players.env_id holds P rows per env.
template <int P>
__device__ __forceinline__ void prefill_ids(char* slots, int64_t slice, int depth, int world,
                                            int n, int id0, int64_t off_env_id,
                                            int64_t off_players) {
  const int64_t total = (int64_t)depth * world * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(i % n);
    const int64_t sg = i / n;
    const int g = (int)(sg % world);
    char* sl = slots + sg * slice;
    reinterpret_cast<int32_t*>(sl + off_env_id)[e] = id0 + g * n + e;
#pragma unroll
    for (int j = 0; j < P; ++j)
      reinterpret_cast<int32_t*>(sl + off_players)[(int64_t)e * P + j] = id0 + g * n + e;
  }
}
__global__ void prefill_ids_kernel(char* slots, int64_t slice, int depth, int world, int n,
                                   int id0, int64_t off_env_id, int64_t off_players) {
  prefill_ids<1>(slots, slice, depth, world, n, id0, off_env_id, off_players);
}
__global__ void prefill_pair_ids_kernel(char* slots, int64_t slice, int depth, int world, int n,
                                        int id0, int64_t off_env_id, int64_t off_players) {
  prefill_ids<2>(slots, slice, depth, world, n, id0, off_env_id, off_players);
}

// Build the per-slot PeerViews from the attached peer bases, copy them to the device and
// write the constant id columns.
int upload_views(epb_pool* p) {
  std::vector<PeerView> v(p->x_depth);
  memset(v.data(), 0, sizeof(PeerView) * v.size());
  for (int slot = 0; slot < p->x_depth; ++slot) {
    PeerView& pv = v[slot];
    pv.world = p->x_world;
    pv.rank = p->x_rank;
    pv.ctl = p->x_ctl();
    pv.ack = reinterpret_cast<const unsigned long long*>(p->x_base + p->x_ack_off);
    pv.timeout_ns = p->x_timeout_ns;
    pv.depth = p->x_depth;
    pv.slot = slot;
    for (int g = 0; g < p->x_world; ++g) {
      pv.slice[g] = p->x_peer[g] + p->x_mine(slot);
      pv.flag[g] = reinterpret_cast<unsigned long long*>(p->x_peer[g] + p->x_data_off) +
                   slot * kMaxPeers + p->x_rank;
    }
    // wire columns: reward, the env keys, the packed common-column word
    int c = 0;
    auto add = [&](int rb, int64_t off) {
      pv.col_rb[c] = rb;
      pv.col_off[c] = off;
      ++c;
    };
    add(p->keys[4].row_bytes, p->keys[4].off);
    for (size_t k = 8; k < p->keys.size(); ++k) add(p->keys[k].row_bytes, p->keys[k].off);
    add(4, p->slab_bytes);
    pv.ncols = c;
  }
  EPB_CUDA(cudaMemcpy(p->x_view(0), v.data(), sizeof(PeerView) * v.size(),
                      cudaMemcpyHostToDevice));
  (p->keys[1].players == 1 ? prefill_ids_kernel : prefill_pair_ids_kernel)
      <<<device_sm_count() * 4, 256, 0, p->stream>>>(
          p->x_base, p->x_slice, p->x_depth, p->x_world, p->N,
          p->cfg.env_id_offset - p->x_rank * p->N, p->keys[0].off, p->keys[1].off);
  EPB_CUDA(cudaGetLastError());
  ++p->launches;
  EPB_CUDA(cudaStreamSynchronize(p->stream));
  p->x_attached = true;
  return EPB_OK;
}

const KindDesc* kind_desc(int kind) {
  for (auto family : {classic_kind, toytext_kind, jumanji_kind, mujoco_kind, pgx_kind})
    if (const KindDesc* d = family(kind)) return d;
  return nullptr;
}

LaunchArgs launch_args(const epb_pool* p, cudaStream_t stream) {
  LaunchArgs a{};
  a.sv = p->sv;
  a.stream = stream;
  a.params = p->params.data();
  return a;
}

// Refill every env's record ring to full on `stream`.
int launch_refill(epb_pool* p, cudaStream_t stream) {
  EPB_CUDA(p->fn.refill(launch_args(p, stream)));
  ++p->launches;
  p->since_refill = 0;
  return EPB_OK;
}

// Launch one batch step on `stream`.  d_action/d_ids are device pointers.
// Record envs (refill policy): chain_k == -1 (direct launches, user-driven captures): a refill
// on the same stream after every `refill_every`-th step launch -- an env consumes at most one
// record per launch, the ring holds rec_q > refill_every.  chain_k == -2: the caller places the
// refill itself (host path: behind the D2H copy; engine-captured chains: on a parallel graph
// branch every refill_every steps, run_chain).  prev_in_slab: LaunchArgs::prev_in_slab.
int launch_batch(epb_pool* p, const void* d_action, const int32_t* d_ids, int n,
                 int force_reset, char* d_slab, cudaStream_t stream, int chain_k = -1,
                 int32_t* wire = nullptr, const void* next_action = nullptr,
                 int prev_in_slab = 0) {
  p->d_last = d_slab;
  p->started = true;
  LaunchArgs a = launch_args(p, stream);
  a.ov = p->slab_view(d_slab);
  p->slab_hi(d_slab, a.env_hi);
  a.ov.wire = wire;
  a.action = d_action;
  a.env_ids = d_ids;
  a.n = n;
  a.force_reset = force_reset;
  a.next_action = next_action;
  a.prev_in_slab = prev_in_slab;
  EPB_CUDA(p->fn.step(a));
  ++p->launches;
  if (p->fn.refill) {
    ++p->since_refill;
    if (chain_k == -1 && p->since_refill >= p->refill_every) return launch_refill(p, stream);
  }
  return EPB_OK;
}

// Host path shared by send and reset.
int host_submit(epb_pool* p, const void* action, const int32_t* env_ids, int n,
                int force_reset) {
  if (n <= 0 || n > p->N) return fail(EPB_ERR_INVALID, "batch rows must be in [1, num_envs]");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  const int f = p->stage_flip;
  p->stage_flip ^= 1;
  // the staging pair alternates; wait until the copy that last used this half is done
  EPB_CUDA(cudaEventSynchronize(p->h_stage_ev[f]));
  // The action goes first: its staging copy and H2D are on the critical path of the step,
  // and the env-id check below (a 4N-byte compare) then runs while the copy is in flight.
  if (!force_reset) {
    if (!action) return fail(EPB_ERR_INVALID, "action is NULL");
    size_t bytes = (size_t)p->act.row_bytes * n;
    memcpy(p->h_action[f], action, bytes);
    EPB_CUDA(cudaMemcpyAsync(p->d_action, p->h_action[f], bytes, cudaMemcpyHostToDevice,
                             p->stream));
  }
  bool identity = (n == p->N);
  if (env_ids) {
    // fast path: the usual sync-mode call passes env_id == arange(N) (python/envpool.py
    // all_env_ids); one memcmp against a cached arange settles it
    if (identity && memcmp(env_ids, p->arange.data(), sizeof(int32_t) * n) == 0) {
      // identity gather, nothing to upload
    } else {
      bool ok = true;
      identity = false;
      const unsigned un = (unsigned)p->N;
      for (int i = 0; i < n; ++i) ok &= (unsigned)env_ids[i] < un;
      if (!ok) {
        cudaEventRecord(p->h_stage_ev[f], p->stream);  // the action copy may still be in flight
        return fail(EPB_ERR_INVALID, "env_id out of range");
      }
    }
  } else if (n != p->N) {
    identity = false;  // rows 0..n-1 of a partial batch: ids are 0..n-1
  }
  const int32_t* d_ids = nullptr;
  if (!identity) {
    if (env_ids) {
      memcpy(p->h_ids[f], env_ids, sizeof(int32_t) * n);
    } else {
      for (int i = 0; i < n; ++i) p->h_ids[f][i] = i;
    }
    EPB_CUDA(cudaMemcpyAsync(p->d_ids, p->h_ids[f], sizeof(int32_t) * n,
                             cudaMemcpyHostToDevice, p->stream));
    d_ids = p->d_ids;
  }
  EPB_CUDA(cudaEventRecord(p->h_stage_ev[f], p->stream));
  // the step kernel alone; the refill of the records it consumed goes BEHIND the D2H copy
  // (the caller waits for the copy, not for the refill)
  int rc = launch_batch(p, p->d_action, d_ids, n, force_reset, p->d_slab, p->stream, -2);
  if (rc != EPB_OK) return rc;
  void* slab = nullptr;
  bool ids_ok = false;
  rc = get_slab(p, &slab, &ids_ok);
  if (rc != EPB_OK) return rc;
  if (n == p->N && identity) {
    // the id columns of a full identity batch are constants the pinned slab already holds
    if (!ids_ok) {
      fill_id_columns(p, slab);
      set_ids_ok(p, slab, true);
    }
    const int64_t from = p->keys[2].off;
    EPB_CUDA(cudaMemcpyAsync(static_cast<char*>(slab) + from, p->d_slab + from,
                             (size_t)(p->slab_bytes - from), cudaMemcpyDeviceToHost,
                             p->stream));
  } else {
    if (ids_ok) set_ids_ok(p, slab, false);
    for (const Key& k : p->keys) {
      EPB_CUDA(cudaMemcpyAsync(static_cast<char*>(slab) + k.off, p->d_slab + k.off,
                               (size_t)k.row_bytes * n, cudaMemcpyDeviceToHost, p->stream));
    }
  }
  cudaEvent_t ev;
  rc = get_event(p, &ev);
  if (rc != EPB_OK) return rc;
  EPB_CUDA(cudaEventRecord(ev, p->stream));
  {
    std::lock_guard<std::mutex> lk(p->mu);
    p->pending.push_back(Pending{slab, n, 0, ev, false});
    p->leases.emplace_back(slab, 1);  // the queue's own reference
  }
  if (p->fn.refill && p->since_refill >= p->refill_every) return launch_refill(p, p->stream);
  return EPB_OK;
}

}  // namespace

extern "C" {

const char* epb_last_error(void) { return g_err.c_str(); }
int epb_abi_version(void) { return EPB_ABI_VERSION; }

int epb_create(int kind, const epb_config* cfg, epb_pool** out) {
  if (!cfg || !out) return fail(EPB_ERR_INVALID, "null argument");
  const KindDesc* d = kind_desc(kind);
  if (!d) return fail(EPB_ERR_INVALID, "unknown env kind");
  if (cfg->num_envs <= 0) return fail(EPB_ERR_INVALID, "num_envs must be positive");
  // EnvSpec ctor check, envpool/core/env_spec.h:75-80
  if (cfg->batch_size > cfg->num_envs)
    return fail(EPB_ERR_INVALID,
                "It is required that batch_size <= num_envs, got num_envs = " +
                    std::to_string(cfg->num_envs) +
                    ", batch_size = " + std::to_string(cfg->batch_size));
  if (cfg->batch_size < 0) return fail(EPB_ERR_INVALID, "batch_size must be >= 0");
  int ndev = 0;
  EPB_CUDA(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(EPB_ERR_INVALID, "bad device ordinal");
  DeviceGuard guard(cfg->device);
  EPB_CUDA(guard.status);

  const int iopt = cfg->iopt < 0 ? d->default_iopt : cfg->iopt;
  if (d->n_iopts && std::find(d->iopts, d->iopts + d->n_iopts, iopt) == d->iopts + d->n_iopts)
    return fail(EPB_ERR_INVALID, d->iopt_error);

  epb_pool* p = new epb_pool();
  p->kind = kind;
  p->cfg = *cfg;
  p->cfg.env_seed = nullptr;
  p->N = cfg->num_envs;
  p->precision = cfg->precision == EPB_PREC_F32 && !d->fp64_only ? 1 : 0;
  p->real_size = p->precision ? 4 : 8;
  p->NR = d->NR;
  p->NI = d->NI;
  build_keys(p, *d);
  p->fn = d->launch(p->precision, iopt);
  if (d->setup) {
    cudaError_t e = d->setup(*cfg, p->params);
    if (e != cudaSuccess) {
      delete p;
      return fail(EPB_ERR_CUDA, std::string("env setup: ") + cudaGetErrorString(e));
    }
  }
  const int64_t N = p->N;
  auto al = [](int64_t b) { return (b + 255) / 256 * 256; };
  int64_t o_flags = 0;
  int64_t o_idx = o_flags + al(4 * N);
  int64_t o_ist = o_idx + al(4 * N);
  int64_t o_rst = o_ist + al(4 * N * (p->NI > 0 ? p->NI : 1));
  // a kind's configuration words sit where real-valued envs keep rstate
  int64_t o_mt = o_rst + al(d->config_words ? 4 * (int64_t)d->config_words
                                            : (int64_t)p->real_size * N * (p->NR > 0 ? p->NR : 1));
  const bool has_rec = p->fn.refill != nullptr;
  int rec_q = 16;  // records per env; ENVPOOL_B200_REC_Q = 4 | 8 | 16
  if (const char* rq = getenv("ENVPOOL_B200_REC_Q")) {
    int v = atoi(rq);
    if (v == 4 || v == 8 || v == 16) rec_q = v;
  }
  p->refill_every = rec_q / 2;  // <= rec_q - 2: see run_chain for the bound
  if (const char* re = getenv("ENVPOOL_B200_REFILL_EVERY")) {
    int v = atoi(re);
    if (v >= 1 && v <= rec_q - 2) p->refill_every = v;
  }
  int64_t o_rec = o_mt + al(4 * N * kMtN);
  int64_t o_rcons = o_rec + (has_rec ? al((int64_t)p->real_size * N * p->NR * rec_q) : 0);
  int64_t o_rprod = o_rcons + (has_rec ? al(N) : 0);
  p->state_bytes = o_rprod + (has_rec ? al(N) : 0);
  cudaError_t e = cudaMalloc(&p->d_state_blob, (size_t)p->state_bytes);
  if (e == cudaSuccess) e = cudaMemset(p->d_state_blob, 0, (size_t)p->state_bytes);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_slab, (size_t)p->slab_bytes);
  if (e == cudaSuccess) e = cudaMemset(p->d_slab, 0, (size_t)p->slab_bytes);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_action, (size_t)p->act.row_bytes * N);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_ids, 4 * (size_t)N);
  for (int f = 0; f < 2 && e == cudaSuccess; ++f) {
    e = cudaHostAlloc(&p->h_action[f], (size_t)p->act.row_bytes * N, cudaHostAllocDefault);
    if (e == cudaSuccess)
      e = cudaHostAlloc(reinterpret_cast<void**>(&p->h_ids[f]), 4 * (size_t)N,
                        cudaHostAllocDefault);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->h_stage_ev[f], cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaStreamCreate(&p->stream);  // blocking: ordered with the legacy default stream (torch interop)
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->mark_side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->x_side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_mark, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreate(&p->ev_t0);
  if (e == cudaSuccess) e = cudaEventCreate(&p->ev_t1);
  for (int h = 0; h < kMaxDepth && e == cudaSuccess; ++h) {
    e = cudaEventCreateWithFlags(&p->x_ev_step[h], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->x_ev_wait[h], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->x_ev_push[h], cudaEventDisableTiming);
  }
  for (int h = 0; h < 2 && e == cudaSuccess; ++h) {
    e = cudaEventCreateWithFlags(&p->ev_step[h], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_refill[h], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) {
    std::string msg = std::string("device allocation: ") + cudaGetErrorString(e);
    epb_destroy(p);
    return fail(EPB_ERR_CUDA, msg);
  }
  p->batch = cfg->batch_size > 0 ? cfg->batch_size : p->N;
  p->arange.resize(p->N);
  for (int i = 0; i < p->N; ++i) p->arange[i] = i;
  {
    // the first pinned slabs now (cudaHostAlloc costs milliseconds: never inside a step):
    // a sync loop holds two (the batch the caller reads + the one in flight), a pipelined or
    // async one a third; capped at 1 GiB of pinned memory
    int want = (int)((int64_t(1) << 30) / (p->slab_bytes > 0 ? p->slab_bytes : 1));
    want = want > 3 ? 3 : (want < 1 ? 1 : want);
    for (int i = 0; i < want; ++i) {
      void* h = nullptr;
      if (alloc_slab(p, &h) != EPB_OK) {
        std::string msg = g_err;
        epb_destroy(p);
        return fail(EPB_ERR_CUDA, msg);
      }
      p->free_slabs.push_back(h);
    }
  }
  char* blob = static_cast<char*>(p->d_state_blob);
  p->sv.n_envs = p->N;
  p->sv.max_steps = cfg->max_episode_steps > 0 ? cfg->max_episode_steps : INT_MAX;
  p->sv.env_id_offset = cfg->env_id_offset;
  p->sv.iopt = iopt;
  p->sv.flags = reinterpret_cast<int32_t*>(blob + o_flags);
  p->sv.mt_idx = reinterpret_cast<int32_t*>(blob + o_idx);
  p->sv.istate = reinterpret_cast<int32_t*>(blob + o_ist);
  p->sv.rstate = blob + o_rst;
  p->sv.mt = reinterpret_cast<uint32_t*>(blob + o_mt);
  if (has_rec) {
    p->sv.rec = blob + o_rec;
    p->sv.rcons = reinterpret_cast<uint8_t*>(blob + o_rcons);
    p->sv.rprod = reinterpret_cast<uint8_t*>(blob + o_rprod);
    p->sv.rec_q = rec_q;
  }

  // seed on device
  int32_t* d_env_seed = nullptr;
  if (cfg->env_seed) {
    e = cudaMalloc(reinterpret_cast<void**>(&d_env_seed), 4 * (size_t)N);
    if (e == cudaSuccess)
      e = cudaMemcpy(d_env_seed, cfg->env_seed, 4 * (size_t)N, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess) {
    seed_kernel<<<(p->N + 127) / 128, 128, 0, p->stream>>>(p->sv, cfg->seed, d_env_seed);
    e = cudaGetLastError();
    ++p->launches;
  }
  if (e == cudaSuccess && p->fn.refill) {  // the first rec_q records of every env
    e = p->fn.refill(launch_args(p, p->stream));
    ++p->launches;
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(p->stream);
  if (d_env_seed) cudaFree(d_env_seed);
  if (e != cudaSuccess) {
    std::string msg = std::string("seeding: ") + cudaGetErrorString(e);
    epb_destroy(p);
    return fail(EPB_ERR_CUDA, msg);
  }
  // algorithmic bytes per env-step of the single-step kernel (identity env_ids):
  // action + 2 x (flags + env state) + every output column (+ the kind's per-step RNG traffic)
  int b = p->act.row_bytes + 2 * (4 + p->NR * p->real_size + p->NI * 4) + p->fn.extra_step_bytes;
  for (const Key& k : p->keys) b += k.row_bytes;
  p->bytes_per_step = b;
  *out = p;
  return EPB_OK;
}

int epb_destroy(epb_pool* p) {
  if (!p) return EPB_OK;
  DeviceGuard guard(p->cfg.device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  for (Pending& pd : p->pending)
    if (!pd.ready) cudaEventDestroy(pd.ev);
  for (cudaEvent_t ev : p->free_events) cudaEventDestroy(ev);
  for (void* s : p->all_slabs) cudaFreeHost(s);
  for (int f = 0; f < 2; ++f) {
    if (p->h_action[f]) cudaFreeHost(p->h_action[f]);
    if (p->h_ids[f]) cudaFreeHost(p->h_ids[f]);
    if (p->h_stage_ev[f]) cudaEventDestroy(p->h_stage_ev[f]);
  }
  for (auto& g : p->graphs) cudaGraphExecDestroy(g.exec);
  for (int g = 0; g < kMaxPeers; ++g)
    if (p->x_ipc[g] && p->x_peer[g]) cudaIpcCloseMemHandle(p->x_peer[g]);
  if (p->x_base) cudaFree(p->x_base);
  if (p->x_trace) cudaFree(p->x_trace);
  if (p->d_state_blob) cudaFree(p->d_state_blob);
  if (p->d_slab) cudaFree(p->d_slab);
  if (p->d_action) cudaFree(p->d_action);
  if (p->d_ids) cudaFree(p->d_ids);
  for (cudaStream_t* st : {&p->side, &p->mark_side, &p->x_side, &p->x_push[0], &p->x_push[1],
                           &p->x_push[2]}) {
    if (*st) {
      cudaStreamSynchronize(*st);
      cudaStreamDestroy(*st);
    }
  }
  for (cudaEvent_t ev : {p->ev_mark, p->ev_t0, p->ev_t1})
    if (ev) cudaEventDestroy(ev);
  for (int h = 0; h < kMaxDepth; ++h) {
    if (p->x_ev_step[h]) cudaEventDestroy(p->x_ev_step[h]);
    if (p->x_ev_wait[h]) cudaEventDestroy(p->x_ev_wait[h]);
    if (p->x_ev_push[h]) cudaEventDestroy(p->x_ev_push[h]);
  }
  for (int h = 0; h < 2; ++h) {
    if (p->ev_step[h]) cudaEventDestroy(p->ev_step[h]);
    if (p->ev_refill[h]) cudaEventDestroy(p->ev_refill[h]);
  }
  if (p->stream) cudaStreamDestroy(p->stream);
  delete p;
  return EPB_OK;
}

int epb_num_state_keys(const epb_pool* p) { return p ? (int)p->keys.size() : 0; }
int epb_num_envs(const epb_pool* p) { return p ? p->N : 0; }
int64_t epb_slab_bytes(const epb_pool* p) { return p ? p->slab_bytes : 0; }

static void fill_info(const Key& k, epb_key_info* out) {
  out->name = k.name;
  out->dtype = k.dtype;
  out->ndim = k.ndim;
  for (int i = 0; i < 3; ++i) out->shape[i] = k.shape[i];
  out->row_bytes = k.row_bytes;
  out->slab_offset = k.off;
}
int epb_state_key(const epb_pool* p, int k, epb_key_info* out) {
  if (!p || !out || k < 0 || k >= (int)p->keys.size()) return fail(EPB_ERR_INVALID, "bad key index");
  fill_info(p->keys[k], out);
  return EPB_OK;
}
int epb_state_key_players(const epb_pool* p, int k) {
  if (!p || k < 0 || k >= (int)p->keys.size()) return fail(EPB_ERR_INVALID, "bad key index");
  return p->keys[k].players;
}
int epb_action_key(const epb_pool* p, epb_key_info* out) {
  if (!p || !out) return fail(EPB_ERR_INVALID, "null argument");
  fill_info(p->act, out);
  return EPB_OK;
}

int epb_send(epb_pool* p, const void* action, const int32_t* env_ids, int n) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  return host_submit(p, action, env_ids, n, 0);
}
int epb_reset(epb_pool* p, const int32_t* env_ids, int n) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  return host_submit(p, nullptr, env_ids, n, 1);
}

namespace {
// slab reference counting: one reference held by the pending queue while rows remain, one
// per outstanding recv lease.  Caller holds p->mu.
void slab_ref(epb_pool* p, void* slab, int delta) {
  for (size_t i = 0; i < p->leases.size(); ++i) {
    if (p->leases[i].first == slab) {
      p->leases[i].second += delta;
      if (p->leases[i].second <= 0) {
        p->leases.erase(p->leases.begin() + i);
        p->free_slabs.push_back(slab);
      }
      return;
    }
  }
  if (delta > 0) p->leases.emplace_back(slab, delta);
}
}  // namespace

// Sync mode (batch == num_envs): hands out the oldest send/reset as a whole (its n rows,
// partial-id sends included).  Async mode: exactly `batch` rows per call, in submission
// order -- on the GPU every env of a send finishes together, so "the first batch_size envs to
// finish" (state_buffer_queue.h:148-163) is the submission order.
int epb_recv_slab_ex(epb_pool* p, void** slab, int* row0, int* n_rows) {
  if (!p || !slab || !n_rows || !row0) return fail(EPB_ERR_INVALID, "null argument");
  const bool async = p->batch < p->N;
  std::unique_lock<std::mutex> lk(p->mu);
  if (p->pending.empty()) return fail(EPB_ERR_STATE, "recv without an outstanding send/reset");
  auto wait_head = [&](Pending& pd) -> cudaError_t {
    if (pd.ready) return cudaSuccess;
    cudaEvent_t ev = pd.ev;
    lk.unlock();
    cudaError_t e = cudaEventSynchronize(ev);
    lk.lock();
    pd.ready = true;
    p->free_events.push_back(ev);
    return e;
  };
  Pending& head = p->pending.front();
  cudaError_t e = wait_head(head);
  if (e != cudaSuccess) return fail(EPB_ERR_CUDA, std::string("recv: ") + cudaGetErrorString(e));
  const int want = async ? p->batch : head.n - head.row0;
  if (head.n - head.row0 >= want) {
    *slab = head.slab;
    *row0 = head.row0;
    *n_rows = want;
    slab_ref(p, head.slab, +1);
    head.row0 += want;
    if (head.row0 == head.n) {
      slab_ref(p, head.slab, -1);  // queue reference
      p->pending.pop_front();
    }
    return EPB_OK;
  }
  // async batch straddles several sends: assemble it in a fresh slab (host memcpy)
  int have = 0;
  for (const Pending& pd : p->pending) have += pd.n - pd.row0;
  if (have < want) return fail(EPB_ERR_STATE, "recv: fewer than batch_size envs outstanding");
  void* dst = nullptr;
  lk.unlock();
  bool dst_ids_ok = false;
  int rc = get_slab(p, &dst, &dst_ids_ok);
  if (rc == EPB_OK && dst_ids_ok) set_ids_ok(p, dst, false);
  lk.lock();
  if (rc != EPB_OK) return rc;
  int filled = 0;
  while (filled < want) {
    Pending& pd = p->pending.front();
    e = wait_head(pd);
    if (e != cudaSuccess) {
      p->free_slabs.push_back(dst);  // nothing leased yet: hand the assembly slab back
      return fail(EPB_ERR_CUDA, std::string("recv: ") + cudaGetErrorString(e));
    }
    int take = pd.n - pd.row0;
    if (take > want - filled) take = want - filled;
    for (const Key& k : p->keys)
      memcpy(static_cast<char*>(dst) + k.off + (size_t)filled * k.row_bytes,
             static_cast<char*>(pd.slab) + k.off + (size_t)pd.row0 * k.row_bytes,
             (size_t)take * k.row_bytes);
    pd.row0 += take;
    filled += take;
    if (pd.row0 == pd.n) {
      slab_ref(p, pd.slab, -1);
      p->pending.pop_front();
    }
  }
  slab_ref(p, dst, +1);
  *slab = dst;
  *row0 = 0;
  *n_rows = want;
  return EPB_OK;
}
int epb_recv_slab(epb_pool* p, void** slab, int* n_rows) {
  int row0 = 0;
  int rc = epb_recv_slab_ex(p, slab, &row0, n_rows);
  if (rc == EPB_OK && row0 != 0) {
    // plain variant cannot express a row offset: only valid in sync mode
    epb_release_slab(p, *slab);
    return fail(EPB_ERR_STATE, "use epb_recv_slab_ex in async mode");
  }
  return rc;
}
int epb_release_slab(epb_pool* p, void* slab) {
  if (!p || !slab) return fail(EPB_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(p->mu);
  slab_ref(p, slab, -1);
  return EPB_OK;
}
int epb_recv(epb_pool* p, void* const* cols, int* n_rows) {
  void* slab = nullptr;
  int n = 0, row0 = 0;
  int rc = epb_recv_slab_ex(p, &slab, &row0, &n);
  if (rc != EPB_OK) return rc;
  if (cols) {
    for (size_t k = 0; k < p->keys.size(); ++k) {
      if (cols[k]) memcpy(cols[k], static_cast<char*>(slab) + p->keys[k].off +
                                       (size_t)row0 * p->keys[k].row_bytes,
                          (size_t)p->keys[k].row_bytes * n);
    }
  }
  if (n_rows) *n_rows = n;
  return epb_release_slab(p, slab);
}

int epb_step_device(epb_pool* p, const void* d_action, const int32_t* d_env_ids, int n,
                    void* stream) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (n <= 0 || n > p->N) return fail(EPB_ERR_INVALID, "batch rows must be in [1, num_envs]");
  if (!d_action) return fail(EPB_ERR_INVALID, "action is NULL");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  return launch_batch(p, d_action, d_env_ids, n, 0, p->d_slab, s);
}
int epb_reset_device(epb_pool* p, const int32_t* d_env_ids, int n, void* stream) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (n <= 0 || n > p->N) return fail(EPB_ERR_INVALID, "batch rows must be in [1, num_envs]");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  return launch_batch(p, nullptr, d_env_ids, n, 1, p->d_slab, s);
}
int epb_outputs_device(const epb_pool* p, void** d_slab) {
  if (!p || !d_slab) return fail(EPB_ERR_INVALID, "null argument");
  *d_slab = p->d_last ? p->d_last : p->d_slab;
  return EPB_OK;
}

int epb_rollout_device(epb_pool* p, const void* d_actions, int T, void* const* d_cols,
                       void* stream) {
  if (!p || !d_actions || !d_cols) return fail(EPB_ERR_INVALID, "null argument");
  if (T <= 0) return fail(EPB_ERR_INVALID, "T must be positive");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  OutView ov{};
  ov.env_id = static_cast<int32_t*>(d_cols[0]);
  ov.players_id = static_cast<int32_t*>(d_cols[1]);
  ov.elapsed = static_cast<int32_t*>(d_cols[2]);
  ov.done = static_cast<uint8_t*>(d_cols[3]);
  ov.reward = static_cast<float*>(d_cols[4]);
  ov.discount = static_cast<float*>(d_cols[5]);
  ov.step_type = static_cast<int32_t*>(d_cols[6]);
  ov.trunc = static_cast<uint8_t*>(d_cols[7]);
  LaunchArgs a = launch_args(p, s);
  for (size_t k = 8; k < p->keys.size(); ++k)
    (k < 13 ? ov.env[k - 8] : a.env_hi[k - 13]) = d_cols[k];
  ov.t_stride_rows = p->N;
  p->started = true;
  a.ov = ov;
  a.action = d_actions;
  a.n = p->N;
  a.T = T;
  EPB_CUDA(p->fn.rollout(a));
  ++p->launches;
  p->since_refill = 0;  // the rollout kernel leaves every record ring full
  return EPB_OK;
}

namespace {

int exchange_step(epb_pool* p, const void* d_action, cudaStream_t s, int chain_k,
                  const void* next_action, cudaStream_t push_stream = nullptr,
                  cudaEvent_t step_done = nullptr);
int exchange_wait_launch(epb_pool* p, cudaStream_t s);

// The node that the next node captured on `st` would depend on alone: the step just captured.
int captured_tail(cudaStream_t st, cudaGraphNode_t* node) {
  cudaStreamCaptureStatus cs;
  const cudaGraphNode_t* deps = nullptr;
  const cudaGraphEdgeData* data = nullptr;
  size_t n = 0;
  EPB_CUDA(cudaStreamGetCaptureInfo_v3(st, &cs, nullptr, nullptr, &deps, &data, &n));
  *node = n == 1 ? deps[0] : nullptr;
  return EPB_OK;
}

// Before the next step node captured on `st`: its edge from `prev` (the step before it) becomes
// programmatic -- its grid launches while `prev` drains, and griddepcontrol.wait holds every
// access back until `prev` has completed and its stores are visible.  Its other edges (the
// join of a refill branch, of the exchange wait and push branches) are set to full
// dependencies: a launch with the PDL attribute would make those programmatic as well.
int program_step_edge(cudaStream_t st, cudaGraphNode_t prev) {
  cudaStreamCaptureStatus cs;
  const cudaGraphNode_t* deps = nullptr;
  const cudaGraphEdgeData* data = nullptr;
  size_t n = 0;
  EPB_CUDA(cudaStreamGetCaptureInfo_v3(st, &cs, nullptr, nullptr, &deps, &data, &n));
  std::vector<cudaGraphNode_t> nodes(deps, deps + n);
  std::vector<cudaGraphEdgeData> edges(n);  // zero: a full dependency
  for (size_t i = 0; i < n; ++i) {
    if (nodes[i] != prev) continue;
    edges[i].from_port = cudaGraphKernelNodePortProgrammatic;
    edges[i].type = cudaGraphDependencyTypeProgrammatic;
  }
  EPB_CUDA(cudaStreamUpdateCaptureDependencies_v2(st, nodes.data(), edges.data(), n,
                                                  cudaStreamSetCaptureDependencies));
  return EPB_OK;
}

// K consecutive sync steps on `st`, step k reading action row (t0 + k) % T.  `fork` (only
// while capturing) puts the off-critical-path kernels on parallel graph branches:
//   * record envs: one refill on p->side after every refill_every-th step (and after the
//     last), beside the following steps.  Refill j (after step k_j) is awaited by the first
//     step after refill j+1 is launched, i.e. it has refill_every steps to finish.  Between
//     the snapshot refill j works from and the completion of refill j+1 lie at most
//     2 * refill_every steps = at most refill_every consumptions per env (a step that resets
//     is never `done`), so a ring of rec_q >= refill_every + 2 records never runs dry;
//   * exchange chains: wait_derive(k) on p->x_side: step k+1 .. k+D-2 compute and push while
//     the batch of step k is still arriving; step k+D-1 waits for it (its credit needs the
//     local release as well as the peers');
//   * timing marks: ev0 takes the timestamp at which step mark0 became ready, ev1 the
//     completion of step mark1-1 -- recorded on a branch of their own, not in series.  Both
//     hang off a step node by a full edge; step mark0 may launch earlier, but it waits for
//     step mark0-1 to complete, the moment ev0 takes.
// `fork` also makes each step's edge from the step before it programmatic (program_step_edge)
// for the kinds whose step kernel allows it (KindLaunch::programmatic_step): nothing but
// kernel nodes ever sits between two steps on `st`, and every join stays a full dependency, so
// the refill bound above holds as it is.  HalfCheetah's pair kernel keeps plain edges.
int run_chain(epb_pool* p, cudaStream_t st, const ChainKey& c, bool fork, cudaEvent_t ev0,
              cudaEvent_t ev1) {
  const size_t row = (size_t)p->act.row_bytes * p->N;
  const char* base = static_cast<const char*>(c.actions);
  const bool rec = fork && p->fn.refill;
  const bool xfork = fork && c.exchange;
  const int R = p->refill_every;
  int nref = 0;          // refills launched so far in this chain
  bool after_trigger = false;
  const int D = p->x_depth;
  const bool pdl = fork && p->fn.programmatic_step;
  cudaGraphNode_t prev = nullptr;  // pdl: the step node captured last
  auto program_edge = [&]() -> int {
    return pdl && prev ? program_step_edge(st, prev) : EPB_OK;
  };
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  const bool capturing = cap != cudaStreamCaptureStatusNone;
  auto mark = [&](cudaEvent_t ev) -> int {
    if (!fork) {  // in series; inside a capture the timed events are external event nodes
      if (capturing) EPB_CUDA(cudaEventRecordWithFlags(ev, st, cudaEventRecordExternal));
      else EPB_CUDA(cudaEventRecord(ev, st));
      return EPB_OK;
    }
    EPB_CUDA(cudaEventRecord(p->ev_mark, st));
    EPB_CUDA(cudaStreamWaitEvent(p->mark_side, p->ev_mark, 0));
    EPB_CUDA(cudaEventRecordWithFlags(ev, p->mark_side, cudaEventRecordExternal));
    return EPB_OK;
  };
  bool marked = false;
  for (int k = 0; k < c.K; ++k) {
    const char* a = base + row * ((c.t0 + k) % c.T);
    const char* nx = base + row * ((c.t0 + k + 1) % c.T);
    if (ev0 && k == c.mark0) {
      int rc = mark(ev0);
      if (rc != EPB_OK) return rc;
      marked = true;
    }
    if (rec && after_trigger && nref >= 2)  // the refill before the one just launched
      EPB_CUDA(cudaStreamWaitEvent(st, p->ev_refill[(nref - 2) & 1], 0));
    after_trigger = false;
    int rc;
    if (c.exchange) {
      if (xfork && k >= D - 1)
        EPB_CUDA(cudaStreamWaitEvent(st, p->x_ev_wait[(k - (D - 1)) % D], 0));
      if (xfork) {
        // The peer stores leave the step chain: step k only computes (into its local slot
        // k % D); push(k), a copy kernel on a branch of its own, sends the wire columns, and
        // wait_derive(k) follows on the wait branch.  Pipelines beside each other:
        //   steps     step(k) after step(k-1), wait_derive(k-D+1) (run-ahead bound) and
        //             push(k-D) (the slot it overwrites has been sent)
        //   pushes    push(k) after step(k), on push branch k % 3: up to three pushes are in
        //             flight together (per-slot flags and counters keep them apart)
        //   waits     wait_derive(k) after push(k) and wait_derive(k-1)
        // A kernel that stores to a peer cannot complete -- and its successor on the same stream
        // cannot start -- before those stores have drained over NVLink, which takes several
        // times the payload's link time.
        // Round trips cannot be shortened, so they are overlapped.
        if (k >= D) EPB_CUDA(cudaStreamWaitEvent(st, p->x_ev_push[(k - D) % D], 0));
        cudaStream_t ps = p->x_push[k % 3];
        rc = program_edge();
        if (rc != EPB_OK) return rc;
        rc = exchange_step(p, a, st, rec ? -2 : -1, nx, ps, p->x_ev_step[k % D]);
        if (rc != EPB_OK) return rc;
        EPB_CUDA(cudaEventRecord(p->x_ev_push[k % D], ps));
        EPB_CUDA(cudaStreamWaitEvent(p->x_side, p->x_ev_push[k % D], 0));
        rc = exchange_wait_launch(p, p->x_side);
        if (rc != EPB_OK) return rc;
        EPB_CUDA(cudaEventRecord(p->x_ev_wait[k % D], p->x_side));
      } else {
        rc = exchange_step(p, a, st, rec ? -2 : -1, nx);
        if (rc != EPB_OK) return rc;
        rc = exchange_wait_launch(p, st);
        if (rc != EPB_OK) return rc;
      }
    } else {
      rc = program_edge();
      if (rc != EPB_OK) return rc;
      // Step k > 0 follows step k - 1 into the same slab with nothing in between (refills
      // touch only the record rings), so it stores only the common columns that change.
      rc = launch_batch(p, a, nullptr, p->N, 0, p->d_slab, st, rec ? -2 : -1, nullptr, nx,
                        k > 0);
      if (rc != EPB_OK) return rc;
    }
    if (pdl) {
      rc = captured_tail(st, &prev);
      if (rc != EPB_OK) return rc;
    }
    if (rec && ((k % R) == R - 1 || k == c.K - 1)) {
      const int h = nref & 1;
      EPB_CUDA(cudaEventRecord(p->ev_step[h], st));
      EPB_CUDA(cudaStreamWaitEvent(p->side, p->ev_step[h], 0));
      rc = launch_refill(p, p->side);
      if (rc != EPB_OK) return rc;
      EPB_CUDA(cudaEventRecord(p->ev_refill[h], p->side));
      ++nref;
      after_trigger = true;
    }
    if (ev1 && k + 1 == c.mark1) {
      if (xfork) {  // an exchanged step is complete when its batch has arrived
        EPB_CUDA(cudaStreamWaitEvent(p->mark_side, p->x_ev_wait[k % D], 0));
        EPB_CUDA(cudaEventRecordWithFlags(ev1, p->mark_side, cudaEventRecordExternal));
      } else {
        rc = mark(ev1);
        if (rc != EPB_OK) return rc;
      }
    }
  }
  // join every branch
  if (rec && nref > 0)  // refills are serialised on p->side: the last one implies the rest
    EPB_CUDA(cudaStreamWaitEvent(st, p->ev_refill[(nref - 1) & 1], 0));
  if (xfork) EPB_CUDA(cudaStreamWaitEvent(st, p->x_ev_wait[(c.K - 1) % D], 0));
  if (fork && (marked || (ev1 && c.mark1 > 0))) {
    EPB_CUDA(cudaEventRecord(p->ev_mark, p->mark_side));
    EPB_CUDA(cudaStreamWaitEvent(st, p->ev_mark, 0));
  }
  return EPB_OK;
}

int chain_entry(epb_pool* p, const void* d_actions, int T_stream, int t0, int K, int use_graph,
                void* stream, int exchange, int mark0, int mark1, float* ms_out) {
  if (!p || !d_actions) return fail(EPB_ERR_INVALID, "null argument");
  if (T_stream <= 0 || K <= 0 || t0 < 0) return fail(EPB_ERR_INVALID, "bad step-chain shape");
  const bool timed = ms_out != nullptr;
  if (timed && !(0 <= mark0 && mark0 < mark1 && mark1 <= K))
    return fail(EPB_ERR_INVALID, "timing marks must satisfy 0 <= mark0 < mark1 <= K");
  if (exchange) {
    if (!p->x_attached) return fail(EPB_ERR_STATE, "exchange: peers not attached");
    if (p->x_waited != p->x_steps)
      return fail(EPB_ERR_STATE, "exchange chain: an exchanged step has not been waited for");
  }
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  if (exchange && use_graph && !p->x_push[0]) {
    // push branches of the captured exchange chains: created on first use (a pool that never
    // captures one never holds them -- streams map onto a bounded set of hardware queues)
    for (cudaStream_t& ps : p->x_push) EPB_CUDA(cudaStreamCreateWithFlags(&ps, cudaStreamNonBlocking));
  }
  if (p->fn.refill && p->since_refill > 0) {  // chains start from full record rings
    int rc = launch_refill(p, s);
    if (rc != EPB_OK) return rc;
  }
  ChainKey key{d_actions, T_stream, t0, K, timed ? mark0 : -1, timed ? mark1 : -1, exchange,
               exchange ? (int)(p->x_steps % p->x_depth) : 0, s};
  cudaEvent_t ev0 = timed ? p->ev_t0 : nullptr, ev1 = timed ? p->ev_t1 : nullptr;
  if (!use_graph) {
    int rc = run_chain(p, s, key, false, ev0, ev1);
    if (rc != EPB_OK) return rc;
  } else {
    cudaGraphExec_t exec = nullptr;
    for (const auto& g : p->graphs)
      if (g.key == key) exec = g.exec;
    if (!exec) {
      if (p->graphs.size() >= 8) {
        cudaGraphExecDestroy(p->graphs.back().exec);
        p->graphs.pop_back();
      }
      cudaGraph_t g = nullptr;
      EPB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      const int64_t before = p->launches;
      const uint64_t xs = p->x_steps, xw = p->x_waited;
      int rc = run_chain(p, s, key, true, ev0, ev1);
      const int64_t launches = p->launches - before;
      p->launches = before;  // capture records, it does not launch
      p->x_steps = xs;
      p->x_waited = xw;
      p->since_refill = 0;
      cudaError_t e = cudaStreamEndCapture(s, &g);
      if (rc != EPB_OK) {
        if (g) cudaGraphDestroy(g);
        return rc;
      }
      if (e != cudaSuccess)
        return fail(EPB_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
      e = cudaGraphInstantiate(&exec, g, 0);
      cudaGraphDestroy(g);
      if (e != cudaSuccess)
        return fail(EPB_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
      p->graphs.insert(p->graphs.begin(), epb_pool::GraphEntry{exec, key, launches});
    }
    int64_t per = 0;
    for (const auto& g : p->graphs)
      if (g.exec == exec) per = g.launches;
    EPB_CUDA(cudaGraphLaunch(exec, s));
    p->launches += per;
    if (exchange) {
      p->x_steps += (uint64_t)K;
      p->x_waited += (uint64_t)K;
    }
  }
  if (exchange) p->d_last = p->x_base + p->x_mine((int)((p->x_steps - 1) % p->x_depth));
  if (timed) {
    EPB_CUDA(cudaStreamSynchronize(s));
    EPB_CUDA(cudaEventElapsedTime(ms_out, p->ev_t0, p->ev_t1));
  }
  return EPB_OK;
}

}  // namespace

int epb_step_many_device(epb_pool* p, const void* d_actions, int T_stream, int t0, int K,
                         int use_graph, void* stream) {
  return chain_entry(p, d_actions, T_stream, t0, K, use_graph, stream, 0, 0, 0, nullptr);
}
int epb_step_many_timed(epb_pool* p, const void* d_actions, int T_stream, int t0, int K,
                        int mark0, int mark1, int exchange, int use_graph, void* stream,
                        float* ms_out) {
  if (!ms_out) return fail(EPB_ERR_INVALID, "null argument");
  return chain_entry(p, d_actions, T_stream, t0, K, use_graph, stream, exchange, mark0, mark1,
                     ms_out);
}
int epb_step_exchange_many_device(epb_pool* p, const void* d_actions, int T_stream, int t0,
                                  int K, int use_graph, void* stream, void** d_gathered) {
  int rc = chain_entry(p, d_actions, T_stream, t0, K, use_graph, stream, 1, 0, 0, nullptr);
  if (rc == EPB_OK && d_gathered)
    *d_gathered = p->x_base + (int64_t)((p->x_steps - 1) % p->x_depth) * p->x_world * p->x_slice;
  return rc;
}

// ---- peer exchange ---------------------------------------------------------------------
int epb_exchange_init(epb_pool* p, int world, int rank, void* ipc_handle_out) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world)
    return fail(EPB_ERR_INVALID, "exchange: world must be in [1,16] and rank in [0,world)");
  if (p->x_base) return fail(EPB_ERR_STATE, "exchange already initialised");
  static_assert(sizeof(cudaIpcMemHandle_t) == EPB_IPC_HANDLE_BYTES, "IPC handle size");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  if (const char* d = getenv("ENVPOOL_B200_EXCHANGE_DEPTH")) {
    int v = atoi(d);
    if (v >= 2 && v <= kMaxDepth) p->x_depth = v;
  }
  p->x_slice = p->slab_bytes + (((int64_t)4 * p->N + 255) / 256) * 256;
  p->x_data_off = (int64_t)p->x_depth * world * p->x_slice;
  p->x_ack_off = p->x_data_off + 8 * kMaxPeers * kMaxDepth;
  p->x_ctl_off = p->x_ack_off + 8 * kMaxPeers;
  p->x_view_off = p->x_ctl_off + 256;
  p->x_bytes = p->x_view_off + (((int64_t)p->x_depth * sizeof(PeerView) + 255) / 256) * 256;
  EPB_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->x_base), (size_t)p->x_bytes));
  EPB_CUDA(cudaMemset(p->x_base, 0, (size_t)p->x_bytes));
  EPB_CUDA(cudaDeviceSynchronize());
  p->x_world = world;
  p->x_rank = rank;
  p->x_peer[rank] = p->x_base;
  if (const char* to = getenv("ENVPOOL_B200_EXCHANGE_TIMEOUT_S")) {
    double sec = atof(to);
    if (sec > 0) p->x_timeout_ns = (long long)(sec * 1e9);
  }
  {
    ExchangeCtl c{};
    for (int sl = 0; sl < p->x_depth; ++sl) c.slot_step[sl] = (unsigned long long)sl;
    const char* tr = getenv("ENVPOOL_B200_EXCHANGE_TRACE");
    if (tr && tr[0] == '1' && !p->x_trace) {
      p->x_trace_steps = 1 << 16;
      EPB_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->x_trace),
                          (size_t)p->x_trace_steps * 8 * sizeof(long long)));
      EPB_CUDA(cudaMemset(p->x_trace, 0, (size_t)p->x_trace_steps * 8 * sizeof(long long)));
    }
    c.trace = p->x_trace;
    c.trace_steps = p->x_trace_steps;
    static_assert(sizeof(ExchangeCtl) <= 256, "ctl block is 256 bytes");
    EPB_CUDA(cudaMemcpy(p->x_base + p->x_ctl_off, &c, sizeof(c), cudaMemcpyHostToDevice));
  }
  if (world == 1) {
    int rc = upload_views(p);
    if (rc != EPB_OK) return rc;
  }
  if (ipc_handle_out) {
    cudaIpcMemHandle_t h;
    EPB_CUDA(cudaIpcGetMemHandle(&h, p->x_base));
    memcpy(ipc_handle_out, &h, sizeof(h));
  }
  return EPB_OK;
}
int epb_exchange_base(const epb_pool* p, void** base, int64_t* bytes) {
  if (!p || !base) return fail(EPB_ERR_INVALID, "null argument");
  if (!p->x_base) return fail(EPB_ERR_STATE, "exchange not initialised");
  *base = p->x_base;
  if (bytes) *bytes = p->x_bytes;
  return EPB_OK;
}
int64_t epb_exchange_slice_bytes(const epb_pool* p) { return p ? p->x_slice : 0; }
int epb_exchange_depth(const epb_pool* p) { return p ? p->x_depth : 0; }
int epb_exchange_attach(epb_pool* p, void* const* peer_bases) {
  if (!p || !peer_bases) return fail(EPB_ERR_INVALID, "null argument");
  if (!p->x_base) return fail(EPB_ERR_STATE, "exchange not initialised");
  for (int g = 0; g < p->x_world; ++g) {
    if (g == p->x_rank) continue;
    if (!peer_bases[g]) return fail(EPB_ERR_INVALID, "exchange: null peer base");
    p->x_peer[g] = static_cast<char*>(peer_bases[g]);
  }
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  return upload_views(p);
}
int epb_exchange_attach_ipc(epb_pool* p, const void* ipc_handles) {
  if (!p || !ipc_handles) return fail(EPB_ERR_INVALID, "null argument");
  if (!p->x_base) return fail(EPB_ERR_STATE, "exchange not initialised");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  for (int g = 0; g < p->x_world; ++g) {
    if (g == p->x_rank || p->x_ipc[g]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const char*>(ipc_handles) + (size_t)g * sizeof(h), sizeof(h));
    void* ptr = nullptr;
    EPB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    p->x_peer[g] = static_cast<char*>(ptr);
    p->x_ipc[g] = true;
  }
  return upload_views(p);
}

namespace {

// One exchanged step on `s`: the step kernel writes slot[t % D][rank] of the local allocation,
// then push_kernel -- on `push_stream` if given, else on `s` -- checks the credit (slot t % D
// released everywhere), forwards the wire columns and publishes.
int exchange_step(epb_pool* p, const void* d_action, cudaStream_t s, int chain_k,
                  const void* next_action, cudaStream_t push_stream, cudaEvent_t step_done) {
  const int D = p->x_depth;
  const uint64_t t = p->x_steps;
  // the credit of step t needs this rank's own release of step t - D, which its wait for
  // step t - D + 1 publishes: that wait must at least have been enqueued
  if (t + 2 > p->x_waited + (uint64_t)D)
    return fail(EPB_ERR_STATE,
                "exchange: too many exchanged steps without epb_exchange_wait (at most "
                "depth - 1 may be outstanding)");
  const int slot = (int)(t % D);
  char* mine = p->x_base + p->x_mine(slot);
  int32_t* wire = reinterpret_cast<int32_t*>(mine + p->slab_bytes);
  const int force = d_action ? 0 : 1;
  int rc = launch_batch(p, d_action, nullptr, p->N, force, mine, s, chain_k, wire, next_action);
  if (rc != EPB_OK) return rc;
  if (push_stream) {  // the copy kernel goes on the caller's side branch, behind this step
    EPB_CUDA(cudaEventRecord(step_done, s));
    EPB_CUDA(cudaStreamWaitEvent(push_stream, step_done, 0));
    s = push_stream;
  }
  // CTAs of the copy kernel: eight 16-byte units per thread (two passes of four), at most 8
  // CTAs per SM.  Every CTA ends in a system-scope fence, so fewer, fuller CTAs make the
  // fence phase cheaper.  ENVPOOL_B200_PUSH_CTAS overrides.
  static const int64_t cta_cap = [] {
    const char* e = getenv("ENVPOOL_B200_PUSH_CTAS");
    const int v = e ? atoi(e) : 0;
    return (int64_t)(v > 0 ? v : device_sm_count() * 8);
  }();
  // reward + the packed word
  int64_t n16 = ((int64_t)p->N * p->keys[4].row_bytes + 15) / 16 + ((int64_t)p->N * 4 + 15) / 16;
  for (size_t k = 8; k < p->keys.size(); ++k)
    n16 += ((int64_t)p->N * p->keys[k].row_bytes + 15) / 16;
  int64_t blocks = (n16 + 2047) / 2048;
  if (blocks > cta_cap) blocks = cta_cap;
  if (blocks < 1) blocks = 1;
  push_kernel<<<(unsigned)blocks, 256, 0, s>>>(p->x_view(slot), p->N);
  EPB_CUDA(cudaGetLastError());
  ++p->launches;
  ++p->x_steps;
  return EPB_OK;
}

// The wait for the oldest exchanged step that has not been waited for (step u = x_waited).
int exchange_wait_launch(epb_pool* p, cudaStream_t s) {
  WaitArgs a{};
  a.data_flag = reinterpret_cast<const unsigned long long*>(p->x_base + p->x_data_off);
  for (int g = 0; g < p->x_world; ++g)
    a.ack_dst[g] =
        reinterpret_cast<unsigned long long*>(p->x_peer[g] + p->x_ack_off) + p->x_rank;
  a.slots = p->x_base;
  a.slice = p->x_slice;
  a.wire_off = p->slab_bytes;
  a.off_elapsed = p->keys[2].off;
  a.off_done = p->keys[3].off;
  a.off_discount = p->keys[5].off;
  a.off_step_type = p->keys[6].off;
  a.off_trunc = p->keys[7].off;
  a.ctl = p->x_ctl();
  a.timeout_ns = p->x_timeout_ns;
  a.world = p->x_world;
  a.rank = p->x_rank;
  a.depth = p->x_depth;
  a.n = p->N;
  // CTAs per peer slice: one quad of envs per thread if the GPU has room (2 CTAs per SM over
  // all peers), never fewer than 16
  int cap = (2 * device_sm_count()) / (p->x_world > 1 ? p->x_world - 1 : 1);
  if (cap < 16) cap = 16;
  int per_peer = (p->N / 4 + 255) / 256;
  if (per_peer > cap) per_peer = cap;
  if (per_peer < 1) per_peer = 1;
  (p->keys[5].players == 1 ? wait_derive_kernel : wait_derive_pair_kernel)
      <<<dim3(per_peer, p->x_world), 256, 0, s>>>(a);
  EPB_CUDA(cudaGetLastError());
  ++p->launches;
  ++p->x_waited;
  return EPB_OK;
}

}  // namespace

int epb_step_exchange_device(epb_pool* p, const void* d_action, void* stream) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (!p->x_attached) return fail(EPB_ERR_STATE, "exchange: peers not attached");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  return exchange_step(p, d_action, s, -1, nullptr);
}
int epb_exchange_wait(epb_pool* p, void* stream, void** d_gathered) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (!p->x_attached || p->x_waited >= p->x_steps)
    return fail(EPB_ERR_STATE, "exchange: no exchanged step is waiting to be received");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : p->stream;
  const int slot = (int)(p->x_waited % p->x_depth);
  int rc = exchange_wait_launch(p, s);
  if (rc != EPB_OK) return rc;
  if (d_gathered) *d_gathered = p->x_base + (int64_t)slot * p->x_world * p->x_slice;
  return EPB_OK;
}
int epb_exchange_trace(epb_pool* p, int64_t* out, int64_t steps) {
  if (!p || !p->x_base || !p->x_trace) return fail(EPB_ERR_STATE, "exchange trace is off");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  if (steps > p->x_trace_steps) steps = p->x_trace_steps;
  EPB_CUDA(cudaMemcpy(out, p->x_trace, (size_t)steps * 8 * sizeof(long long),
                      cudaMemcpyDeviceToHost));
  return EPB_OK;
}
int epb_exchange_status(epb_pool* p, int64_t* steps_pushed, int* timed_out) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (!p->x_base) return fail(EPB_ERR_STATE, "exchange not initialised");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  ExchangeCtl c{};
  EPB_CUDA(cudaMemcpy(&c, p->x_base + p->x_ctl_off, sizeof(c), cudaMemcpyDeviceToHost));
  if (steps_pushed) *steps_pushed = (int64_t)c.seq;
  if (timed_out) *timed_out = c.error;
  return EPB_OK;
}

int epb_sync(epb_pool* p) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaStreamSynchronize(p->stream));
  return EPB_OK;
}
void* epb_stream(epb_pool* p) { return p ? static_cast<void*>(p->stream) : nullptr; }

int64_t epb_state_bytes(const epb_pool* p) { return p ? p->state_bytes : 0; }
int epb_state_layout(const epb_pool* p, int64_t* out) {
  if (!p || !out) return fail(EPB_ERR_INVALID, "null argument");
  const char* blob = static_cast<const char*>(p->d_state_blob);
  out[0] = reinterpret_cast<const char*>(p->sv.flags) - blob;
  out[1] = reinterpret_cast<const char*>(p->sv.mt_idx) - blob;
  out[2] = reinterpret_cast<const char*>(p->sv.istate) - blob;
  out[3] = static_cast<const char*>(p->sv.rstate) - blob;
  out[4] = reinterpret_cast<const char*>(p->sv.mt) - blob;
  out[5] = p->NI;
  out[6] = p->NR;
  out[7] = p->real_size;
  out[8] = p->sv.rec ? static_cast<const char*>(p->sv.rec) - blob : -1;
  out[9] = p->sv.rcons ? reinterpret_cast<const char*>(p->sv.rcons) - blob : -1;
  out[10] = p->sv.rprod ? reinterpret_cast<const char*>(p->sv.rprod) - blob : -1;
  out[11] = p->sv.rec_q;
  return EPB_OK;
}
int epb_state_export(epb_pool* p, void* host_dst) {
  if (!p || !host_dst) return fail(EPB_ERR_INVALID, "null argument");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaStreamSynchronize(p->stream));
  EPB_CUDA(cudaMemcpy(host_dst, p->d_state_blob, (size_t)p->state_bytes, cudaMemcpyDeviceToHost));
  return EPB_OK;
}
int epb_state_import(epb_pool* p, const void* host_src) {
  if (!p || !host_src) return fail(EPB_ERR_INVALID, "null argument");
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaStreamSynchronize(p->stream));
  EPB_CUDA(cudaMemcpy(p->d_state_blob, host_src, (size_t)p->state_bytes, cudaMemcpyHostToDevice));
  p->imported = true;
  if (p->fn.refill) {
    // a blob may carry a ring that is not full (a hand-edited RNG table wants its next resets
    // drawn from that table: rprod = rcons empties the ring): fill it now
    int rc = launch_refill(p, p->stream);
    if (rc != EPB_OK) return rc;
    EPB_CUDA(cudaStreamSynchronize(p->stream));
  }
  return EPB_OK;
}

namespace {
// 8 independent DFMA chains per thread: the fp64 FMA pipe's sustained rate (the denominator of
// HalfCheetah's compute roofline, measured rather than taken from a data sheet).
__global__ void __launch_bounds__(256) fp64_peak_kernel(double* out, int iters, double seed) {
  double a0 = seed + threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4,
         a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double m = 0.999999, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  double r = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
  if (r == 12345.678) out[0] = r;  // never true: keeps the chains alive
}
}  // namespace

int epb_fp64_peak_gflops(int device, double* gflops_out) {
  if (!gflops_out) return fail(EPB_ERR_INVALID, "null argument");
  DeviceGuard guard(device);
  EPB_CUDA(guard.status);
  double* d = nullptr;
  EPB_CUDA(cudaMalloc(reinterpret_cast<void**>(&d), 8));
  cudaEvent_t e0, e1;
  EPB_CUDA(cudaEventCreate(&e0));
  EPB_CUDA(cudaEventCreate(&e1));
  const int grid = device_sm_count() * 8, iters = 1 << 14;
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    EPB_CUDA(cudaEventRecord(e0, 0));
    fp64_peak_kernel<<<grid, 256>>>(d, iters, 1.0 + rep);
    EPB_CUDA(cudaEventRecord(e1, 0));
    EPB_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    EPB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d);
  *gflops_out = 2.0 * 8.0 * iters * 256.0 * grid / (best * 1e-3) / 1e9;
  return EPB_OK;
}

int64_t epb_hc_model(void* dst, int64_t cap) { return mjc_model_blob(dst, cap); }
int epb_hc_pair_rows(const epb_pool* p, int n) {
  if (!p || p->kind != EPB_HALF_CHEETAH || n <= 0 || n > p->N) return 0;
  DeviceGuard guard(p->cfg.device);  // the SM count is read from the pool's device
  return guard.status == cudaSuccess ? mjc_pair_rows(n) : 0;
}
int epb_game2048_boards(epb_pool* p, const int32_t* initial16, const int32_t* replay512) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (p->kind != EPB_GAME2048) return fail(EPB_ERR_INVALID, "not a Game2048 pool");
  if (p->started)
    return fail(EPB_ERR_STATE, "Game2048 boards must be set before the pool's first reset");
  std::vector<uint32_t> words;
  int32_t iopt = p->sv.iopt;
  if (const char* err = game2048_config(initial16, replay512, words, iopt))
    return fail(EPB_ERR_INVALID, err);
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaMemcpy(p->sv.rstate, words.data(), 4 * words.size(), cudaMemcpyHostToDevice));
  p->sv.iopt = iopt;
  return EPB_OK;
}
int epb_minesweeper_config(epb_pool* p, const int32_t* mines100, const int32_t* replay_boards3200,
                           const float* replay_rewards32, const uint8_t* replay_done32) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (p->kind != EPB_MINESWEEPER) return fail(EPB_ERR_INVALID, "not a Minesweeper pool");
  if (p->started)
    return fail(EPB_ERR_STATE, "Minesweeper configuration must be set before the pool's first reset");
  std::vector<uint32_t> words;
  if (const char* err = minesweeper_config(mines100, replay_boards3200, replay_rewards32,
                                           replay_done32, words))
    return fail(EPB_ERR_INVALID, err);
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaMemcpy(p->sv.rstate, words.data(), 4 * words.size(), cudaMemcpyHostToDevice));
  return EPB_OK;
}
int epb_go_config(epb_pool* p, double komi, int32_t max_terminal_steps) {
  if (!p) return fail(EPB_ERR_INVALID, "null pool");
  if (p->kind != EPB_GO_9X9 && p->kind != EPB_GO_13X13 && p->kind != EPB_GO_19X19)
    return fail(EPB_ERR_INVALID, "not a Go pool");
  if (p->started || p->imported)
    return fail(EPB_ERR_STATE, "Go configuration must be set before the pool's first reset, "
                               "step, rollout or state import");
  std::vector<uint32_t> words;
  if (const char* err = go_config(p->kind, komi, max_terminal_steps, words))
    return fail(EPB_ERR_INVALID, err);
  DeviceGuard guard(p->cfg.device);
  EPB_CUDA(guard.status);
  EPB_CUDA(cudaMemcpy(p->sv.rstate, words.data(), 4 * words.size(), cudaMemcpyHostToDevice));
  return EPB_OK;
}
int64_t epb_launch_count(const epb_pool* p) { return p ? p->launches : 0; }
int epb_bytes_per_env_step(const epb_pool* p) { return p ? p->bytes_per_step : 0; }

}  // extern "C"
