// gb_peer.cu -- the fused multi-GPU result exchange (peer slabs over CUDA IPC, DESIGN.md §8): the gb_peer_slab_* entry
// points, gb_sweep_attach_peer_slab and the two exchange kernels.  The sweep kernels' side of it, the pair_push of their
// epilogue, reads PeerPush and the slab regions of gb_internal.cuh.
#include "gb_internal.cuh"

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

// completion flags of the fused exchange: one thread per rank publishes this rank's step to that peer, then waits for the
// peer's flag.  The preceding sweep kernel has completed (stream order), so all its peer stores have been performed.
struct PeerFlags { unsigned* flags[GB_MAX_PEERS]; };
__global__ void k_peer_signal_wait(PeerFlags pf, int world, int rank, unsigned step, int* timeout) {
  const int t = threadIdx.x;
  if (t >= world) return;
  __threadfence_system();
  volatile unsigned* remote = pf.flags[t] + rank;
  *remote = step;
  __threadfence_system();
  volatile unsigned* mine = pf.flags[rank] + t;
  const long long t0 = clock64();
  while ((int)(*mine - step) < 0) {
    __nanosleep(200);
    if (clock64() - t0 > 4000000000ll) { *timeout = 1; break; }  // ~2 s: a peer died; do not hold the GPU
  }
  __threadfence_system();
}

// Deferred exchange: the four CTAs of peer p copy this rank's finished rows (written by the sweep into the local buffer of the step
// parity) into peer p's buffer -- 128-bit stores through the IPC mapping, ~164 KB per peer at 8 ranks -- then publishes this
// rank's step to that peer and waits for the peer's flag.  The CTAs are independent (one per peer): no ordering between them.
// Why not from the sweep's epilogue (GB_PEER_PUSH=fused, the round-1 design): stores to peer memory issued from all the busy
// SMs slow the sweep down at 8 ranks (against the same shard without the peer stores) while the whole exchange is ~1 MB per rank
// and step.
struct PeerExchange {
  float* dst[GB_MAX_PEERS];   // every rank's buffer of the step parity, as mapped here
  unsigned* flags[GB_MAX_PEERS];
  const float* src;           // this rank's buffer of the step parity
  const int* my_pairs;
  int num_my_pairs;
  unsigned* arrivals;         // [world] CTA arrival counters (self-cleaning)
};
constexpr int kExchangeCtasPerPeer = 4;
constexpr int kExchangeThreads = 512;
__global__ void __launch_bounds__(kExchangeThreads) k_peer_exchange(PeerExchange px, int world, int rank, unsigned step, int* timeout) {
  const int p = blockIdx.x / kExchangeCtasPerPeer, c = blockIdx.x % kExchangeCtasPerPeer;
  if (p != rank) {
    float4* __restrict__ dst = reinterpret_cast<float4*>(px.dst[p]);
    const float4* __restrict__ src = reinterpret_cast<const float4*>(px.src);
    constexpr int kVec = GB_SLAB_STRIDE / 4;
    const int total = px.num_my_pairs * kVec;
    const int stride = kExchangeCtasPerPeer * kExchangeThreads;
    // four independent 16-byte loads in flight per thread: the copy is latency-, not bandwidth-bound (~1 MB per rank and step)
    for (int e0 = c * kExchangeThreads + threadIdx.x; e0 < total; e0 += 4 * stride) {
      float4 v[4];
      size_t at[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int e = min(e0 + u * stride, total - 1);
        at[u] = (size_t)px.my_pairs[e / kVec] * kVec + (size_t)(e % kVec);
        v[u] = __ldcg(&src[at[u]]);
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        if (e0 + u * stride < total) dst[at[u]] = v[u];
    }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x != 0) return;
  // the last of this peer's CTAs publishes the flag and waits for the peer's
  const unsigned arrived = atomicAdd(&px.arrivals[p], 1u);
  if (arrived != (unsigned)kExchangeCtasPerPeer - 1u) return;
  px.arrivals[p] = 0u;
  __threadfence_system();
  volatile unsigned* remote = px.flags[p] + rank;
  *remote = step;
  volatile unsigned* mine = px.flags[rank] + p;
  const long long t0 = clock64();
  while ((int)(*mine - step) < 0) {
    __nanosleep(100);
    if (clock64() - t0 > 4000000000ll) { *timeout = 1; break; }  // ~2 s: a peer died; do not hold the GPU
  }
  __threadfence_system();
}

static gb_status launch_peer_signal_wait(gb_peer_slab* ps) {
  const gb_peer_regions mine = gb_peer_regions_of(ps, ps->rank);
  if (ps->deferred) {
    PeerExchange px;
    memset(&px, 0, sizeof(px));
    for (int p = 0; p < ps->world; p++) {
      const gb_peer_regions r = gb_peer_regions_of(ps, p);
      px.dst[p] = r.buf[ps->parity];
      px.flags[p] = r.flags;
    }
    px.src = mine.buf[ps->parity];
    px.my_pairs = ps->d_my_pairs;
    px.num_my_pairs = ps->num_my_pairs;
    px.arrivals = mine.arrivals;
    return gb_launch(ps->ctx, "k_peer_exchange", k_peer_exchange, ps->world * kExchangeCtasPerPeer, kExchangeThreads, 0, px, ps->world, ps->rank, ps->step, mine.timeout);
  }
  PeerFlags pf;
  memset(&pf, 0, sizeof(pf));
  for (int p = 0; p < ps->world; p++) pf.flags[p] = gb_peer_regions_of(ps, p).flags;
  return gb_launch(ps->ctx, "k_peer_signal_wait", k_peer_signal_wait, 1, 32, 0, pf, ps->world, ps->rank, ps->step, mine.timeout);
}

// The pinned block of the fetches: the rows of the completed buffer, then its timeout word.
struct PeerFetch {
  float* rows;  // num_pairs x GB_SLAB_STRIDE
  int* timeout;
};
static PeerFetch peer_fetch_layout(Carver& cv, size_t num_pairs) {
  PeerFetch b;
  b.rows = cv.take<float>(num_pairs * GB_SLAB_STRIDE);
  b.timeout = cv.take<int>(1);
  return b;
}

static void peer_slab_free(gb_peer_slab* ps) {
  gb_ctx* ctx = ps->ctx;
  {
    GB_LOCK(ctx);
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (int p = 0; p < ps->world; p++)
      if (ps->opened[p]) cudaIpcCloseMemHandle(ps->peer[p]);
    if (ps->local) cudaFree(ps->local);
    if (ps->d_my_pairs) cudaFree(ps->d_my_pairs);
    if (ps->h_pinned) cudaFreeHost(ps->h_pinned);
    delete ps;
  }
  ctx_release(ctx);  // outside the lock: it may delete the context
}

extern "C" gb_status gb_peer_slab_create(gb_ctx* ctx, size_t num_pairs, int world, int rank, gb_peer_slab** out) {
  GB_REQUIRE(ctx && out, "null argument");
  GB_REQUIRE(world >= 1 && world <= GB_MAX_PEERS && rank >= 0 && rank < world, "world must be 1..8 and rank < world");
  GB_REQUIRE(num_pairs > 0, "num_pairs must be positive");
  *out = nullptr;
  GB_ENTER(ctx);
  gb_owned<gb_peer_slab> ps(new (std::nothrow) gb_peer_slab(), peer_slab_free);
  if (!ps) return GB_ERR_INTERNAL;
  ctx_retain(ctx);
  ps->ctx = ctx; ps->num_pairs = num_pairs; ps->world = world; ps->rank = rank;
  ps->connected = (world == 1);
  // fused: the sweep's epilogue stores every finished row straight into all peers; deferred: rows go to the local buffer and
  // the exchange kernel pushes them (see k_peer_exchange).  The peer stores' cost to the sweep grows with the
  // rank count faster than the exchange kernel's extra time -> fused up to 4 ranks, deferred above.  GB_PEER_PUSH=fused|deferred forces one.
  {
    const char* e = getenv("GB_PEER_PUSH");
    ps->deferred = world > 4;
    if (e && !strcmp(e, "fused")) ps->deferred = false;
    if (e && !strcmp(e, "deferred")) ps->deferred = true;
  }
  Carver size;
  gb_peer_layout(size, num_pairs, world);
  GB_CUDA(cudaMalloc((void**)&ps->local, size.off));
  ps->peer[rank] = ps->local;
  GB_CUDA(cudaMemsetAsync(ps->local, 0, size.off, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  Carver fetch;
  peer_fetch_layout(fetch, num_pairs);
  GB_CUDA(cudaMallocHost((void**)&ps->h_pinned, fetch.off));
  *out = ps.release();
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_export(gb_peer_slab* ps, void* handle) {
  GB_REQUIRE(ps && handle, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == GB_IPC_HANDLE_BYTES, "IPC handle size");
  GB_ENTER(ps->ctx);
  cudaIpcMemHandle_t h;
  GB_CUDA(cudaIpcGetMemHandle(&h, ps->local));
  memcpy(handle, &h, sizeof(h));
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_connect(gb_peer_slab* ps, const void* handles) {
  GB_REQUIRE(ps && handles, "null argument");
  GB_ENTER(ps->ctx);
  for (int p = 0; p < ps->world; p++) {
    if (p == ps->rank || ps->opened[p]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + (size_t)p * GB_IPC_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    GB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    ps->peer[p] = (char*)ptr;
    ps->opened[p] = true;
  }
  ps->connected = true;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_destroy(gb_peer_slab* ps) {
  if (ps) peer_slab_free(ps);
  return GB_OK;
}

// Replaces the device block *block (nullptr: none yet; the stream has drained) with a fresh cudaMalloc block of the layout.
// *block is the layout's first array: measuring sets it to nullptr, so it never points at a freed block.
template <typename Layout> static gb_status dev_block_realloc(void** block, Layout&& layout) {
  if (*block) GB_CUDA(cudaFree(*block));
  Carver size;
  layout(size);
  Carver cv;
  GB_CUDA(cudaMalloc((void**)&cv.base, size.off));
  layout(cv);
  return GB_OK;
}

extern "C" gb_status gb_sweep_attach_peer_slab(gb_sweep* s, gb_peer_slab* ps) {
  GB_REQUIRE(s, "null sweep");
  if (!ps) { s->peer = nullptr; return GB_OK; }
  GB_REQUIRE(!s->gicp, "no peer slab can be attached to a GICP sweep");
  GB_REQUIRE(ps->ctx == s->ctx, "peer slab belongs to another context");
  GB_REQUIRE(ps->connected, "connect the peer slab (gb_peer_slab_connect) before attaching it");
  // CSR: global pair id -> this sweep's factor indices
  const size_t P = ps->num_pairs;
  std::vector<int> ptr(P + 1, 0), fac(s->F);
  for (size_t f = 0; f < s->F; f++) {
    GB_REQUIRE(s->h_pair[f] >= 0 && (size_t)s->h_pair[f] < P, "pair index out of range for this peer slab");
    ptr[s->h_pair[f] + 1]++;
  }
  for (size_t k = 0; k < P; k++) ptr[k + 1] += ptr[k];
  std::vector<int> fill(ptr.begin(), ptr.end() - 1);
  for (size_t f = 0; f < s->F; f++) fac[fill[s->h_pair[f]]++] = (int)f;
  // the pairs this sweep owns (one sweep per peer slab): the rows the exchange kernel copies to the peers
  std::vector<int> mine;
  for (size_t k = 0; k < P; k++) if (ptr[k + 1] > ptr[k]) mine.push_back((int)k);
  GB_ENTER(s->ctx);
  GB_CUDA(cudaStreamSynchronize(s->ctx->stream));
  GB_CHECK(dev_block_realloc((void**)&s->d_pair_ptr, [&](Carver& cv) {
    s->d_pair_ptr = cv.take<int>(P + 1);
    s->d_pair_factors = cv.take<int>(std::max<size_t>(1, s->F));
    s->d_pair_done = cv.take<unsigned>(P);
    s->d_peer_tables = cv.take<PeerPush>(2);
  }));
  GB_CHECK(dev_block_realloc((void**)&ps->d_my_pairs, [&](Carver& cv) { ps->d_my_pairs = cv.take<int>(std::max<size_t>(1, mine.size())); }));
  PeerPush tabs[2];
  memset(tabs, 0, sizeof(tabs));
  for (int par = 0; par < 2; par++) {
    if (ps->deferred) {  // the sweep writes this rank's buffer only
      tabs[par].world = 1;
      tabs[par].base[0] = gb_peer_regions_of(ps, ps->rank).buf[par];
    } else {
      tabs[par].world = ps->world;
      for (int p = 0; p < ps->world; p++) tabs[par].base[p] = gb_peer_regions_of(ps, p).buf[par];
    }
    tabs[par].pair_ptr = s->d_pair_ptr; tabs[par].pair_factors = s->d_pair_factors; tabs[par].pair_done = s->d_pair_done;
  }
  GB_CUDA(cudaMemcpy(s->d_peer_tables, tabs, sizeof(tabs), cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemcpy(s->d_pair_ptr, ptr.data(), sizeof(int) * (P + 1), cudaMemcpyHostToDevice));
  if (s->F) GB_CUDA(cudaMemcpy(s->d_pair_factors, fac.data(), sizeof(int) * s->F, cudaMemcpyHostToDevice));
  GB_CUDA(cudaMemset(s->d_pair_done, 0, sizeof(unsigned) * P));
  ps->num_my_pairs = (int)mine.size();
  if (!mine.empty()) GB_CUDA(cudaMemcpy(ps->d_my_pairs, mine.data(), sizeof(int) * mine.size(), cudaMemcpyHostToDevice));
  s->peer = ps;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_signal_wait(gb_peer_slab* ps) {
  GB_REQUIRE(ps, "null peer slab");
  GB_REQUIRE(ps->connected, "gb_peer_slab_connect has not been called");
  GB_ENTER(ps->ctx);
  ps->step++;
  GB_CHECK(launch_peer_signal_wait(ps));
  ps->completed_parity = ps->parity;
  ps->parity ^= 1;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_device_ptr(gb_peer_slab* ps, void** device_ptr) {
  GB_REQUIRE(ps && device_ptr, "null argument");
  *device_ptr = gb_peer_regions_of(ps, ps->rank).buf[ps->completed_parity];
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch_async(gb_peer_slab* ps, const float** host_ptr) {
  GB_REQUIRE(ps, "null peer slab");
  GB_ENTER(ps->ctx);
  const size_t bytes = ps->num_pairs * GB_SLAB_STRIDE * sizeof(float);
  const gb_peer_regions r = gb_peer_regions_of(ps, ps->rank);
  Carver cv{(char*)ps->h_pinned};
  const PeerFetch h = peer_fetch_layout(cv, ps->num_pairs);
  GB_CUDA(cudaMemcpyAsync(h.rows, r.buf[ps->completed_parity], bytes, cudaMemcpyDeviceToHost, ps->ctx->stream));
  GB_CUDA(cudaMemcpyAsync(h.timeout, r.timeout, sizeof(int), cudaMemcpyDeviceToHost, ps->ctx->stream));
  if (host_ptr) *host_ptr = h.rows;
  return GB_OK;
}

extern "C" gb_status gb_peer_slab_fetch(gb_peer_slab* ps, float* host) {
  GB_REQUIRE(ps && host, "null argument");
  GB_ENTER(ps->ctx);
  GB_CHECK(gb_peer_slab_fetch_async(ps, nullptr));
  GB_CUDA(cudaStreamSynchronize(ps->ctx->stream));
  Carver cv{(char*)ps->h_pinned};
  const PeerFetch h = peer_fetch_layout(cv, ps->num_pairs);
  if (*h.timeout) { gb_set_error("peer slab: a peer did not publish its completion flag within the timeout"); return GB_ERR_INTERNAL; }
  memcpy(host, h.rows, ps->num_pairs * GB_SLAB_STRIDE * sizeof(float));
  return GB_OK;
}
