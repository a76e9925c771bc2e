// halo.cu -- one rank of a node-range partition of a single large graph (SURVEY.md 8e; BASELINE config 5).
//
// The reference is single-device; its VarMisuse batches (tasks/varmisuse_task.py:451-538) are what outgrow one GPU.
// Rank r owns the nodes [cuts[r], cuts[r+1]) and every edge whose TARGET it owns, so scatter / softmax / layer norm / GRU
// stay local; the source rows owned by other ranks ("halo") are refreshed once per layer.
//
//   rgnn_halo_plan_create   builds, ON THE DEVICE, the rank-local structure from adjacency lists with GLOBAL node ids:
//                           keeps the edges whose target is owned (order-preserving cub::DeviceSelect), collects the
//                           distinct remote sources (radix sort + unique = the halo list, sorted by global id and therefore
//                           grouped by owner), renumbers (owned nodes first, then halo nodes), and builds the ordinary
//                           rgnn_plan over the local ids, restricted to the owned targets.
//   rgnn_halo_exchange      PULLS the halo rows straight out of the owners' state buffers, which the host has mapped into
//                           this process (CUDA IPC over NVLink / NVSwitch peer access: rgnn_peer_*): ONE kernel per layer,
//                           no packing, no send side, no NCCL call.  The kernel carries its own cross-rank barrier
//                           (system-scope release/acquire flags in peer memory, an epoch counter in device memory so that
//                           the whole layer sequence can be captured into a CUDA graph and replayed).
// Because the exchange is pull-based a rank needs only ITS OWN halo list -- nobody computes what its peers need
// (round 1's host builder did that with np.unique over all edges for every peer).
//
// Training adds the transpose of the pull:
//   rgnn_halo_plan_build_reverse  every rank has published its halo list (owner, row) in peer memory
//                                 (rgnn_halo_plan_attach_grad); each rank reads its peers' lists and builds, ON THE DEVICE,
//                                 a CSR over its owned rows of the (peer, row in that peer's gradient buffer) pairs that
//                                 consumed each row -- radix-sorted by (owned row, peer rank).
//   rgnn_halo_exchange_backward   each rank copies the gradients of its halo rows into its peer-visible gradient buffer;
//                                 after a barrier of its own (separate flags and epoch), every owner computes
//                                 d_own[r] = g_local[r] + sum over the consumers of r in ascending peer rank -- a fixed
//                                 order, no atomics, bit-reproducible.
#include "plan.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <new>
#include <string.h>

struct rgnn_halo_plan {
  int32_t rank = 0, world = 1;
  int32_t lo = 0, n_own = 0, n_halo = 0, n_local = 0;
  int32_t L = 0;
  int64_t cuts[RGNN_MAX_WORLD + 1] = {0};
  int64_t num_edges[RGNN_MAX_EDGE_TYPES] = {0};   // kept edges per type
  int32_t* local_adj[RGNN_MAX_EDGE_TYPES] = {nullptr};   // [E_l, 2] local ids (inside `block`)
  int32_t* halo_global = nullptr;                 // [n_halo] sorted global ids
  int32_t* halo_owner = nullptr;                  // [n_halo]
  int32_t* halo_row = nullptr;                    // [n_halo] row inside the owner's state buffer (= global id - cuts[owner])
  uint32_t* epoch = nullptr;                      // device: number of completed exchanges
  uint32_t* ticket = nullptr;                     // device: CTAs finished in the running exchange
  void* block = nullptr;
  rgnn_plan_t* graph = nullptr;
  // peer memory (rgnn_halo_plan_attach)
  float* peer_state[2][RGNN_MAX_WORLD] = {{nullptr}};
  uint32_t* peer_flags[RGNN_MAX_WORLD] = {nullptr};
  bool attached = false;
  // training (rgnn_halo_plan_attach_grad / rgnn_halo_plan_build_reverse / rgnn_halo_exchange_backward)
  float* peer_grad[2][RGNN_MAX_WORLD] = {{nullptr}};
  uint32_t* peer_grad_flags[RGNN_MAX_WORLD] = {nullptr};
  const int32_t* peer_lists[RGNN_MAX_WORLD] = {nullptr};
  bool grad_attached = false;
  uint32_t* grad_epoch = nullptr;                 // device: completed backward exchanges (not shared with `epoch`)
  uint32_t* grad_ticket = nullptr;
  int64_t n_rev = -1;                             // entries of the reverse index; -1 = not built
  int32_t* rev_off = nullptr;                     // [n_own + 1] CSR over the owned rows
  int32_t* rev_peer = nullptr;                    // [n_rev] consuming rank, ascending within a row
  int32_t* rev_row = nullptr;                     // [n_rev] row of the consumer's gradient buffer (n_own of it + halo index)
  void* rev_block = nullptr;
  cudaStream_t side = nullptr;         // overlapped exchange: the pull kernel runs here, forked from / joined into the caller's stream
  cudaEvent_t ev_fork = nullptr, ev_done = nullptr;
  int device = 0;
  cudaStream_t stream = nullptr;
};

namespace rgnn {
namespace {

struct OwnedTarget {
  int lo, hi;
  __host__ __device__ bool operator()(const int2& e) const { return e.y >= lo && e.y < hi; }
};

constexpr uint32_t HALO_SENTINEL = 0xFFFFFFFFu;

struct KeptTable {
  const int2* adj[RGNN_MAX_EDGE_TYPES];
  int32_t count[RGNN_MAX_EDGE_TYPES];
  int32_t off[RGNN_MAX_EDGE_TYPES];
};

// key of every kept edge: its source's global id when that is remote, else the sentinel.  grid = (ceil(maxE/256), L)
__global__ void halo_keys_kernel(const __grid_constant__ KeptTable t, int lo, int hi, int num_global, uint32_t* __restrict__ keys,
                                 int* __restrict__ err) {
  const int l = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.count[l]) return;
  const int src = t.adj[l][i].x;
  if (src < 0 || src >= num_global) atomicExch(err, 1);
  keys[t.off[l] + i] = (src >= lo && src < hi) || src < 0 || src >= num_global ? HALO_SENTINEL : (uint32_t)src;
}

__global__ void halo_count_kernel(const uint32_t* __restrict__ uniq, const int* __restrict__ num_unique, int* __restrict__ n_halo) {
  const int n = *num_unique;
  *n_halo = (n > 0 && uniq[n - 1] == HALO_SENTINEL) ? n - 1 : n;
}

__device__ __forceinline__ int lower_bound_u32(const uint32_t* a, int n, uint32_t x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct LocalTable { int32_t* adj[RGNN_MAX_EDGE_TYPES]; };

// local ids: owned node g -> g - lo; halo node g -> n_own + position in the sorted halo list
__global__ void halo_renumber_kernel(const __grid_constant__ KeptTable t, const __grid_constant__ LocalTable out, int lo, int hi,
                                     int n_own, const uint32_t* __restrict__ halo, int n_halo) {
  const int l = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.count[l]) return;
  const int2 e = t.adj[l][i];
  int s;
  if (e.x >= lo && e.x < hi) s = e.x - lo;
  else {
    const int pos = lower_bound_u32(halo, n_halo, (uint32_t)e.x);
    s = (pos < n_halo && halo[pos] == (uint32_t)e.x) ? n_own + pos : 0;   // out-of-range ids were flagged; stay memory-safe
  }
  reinterpret_cast<int2*>(out.adj[l])[i] = make_int2(s, e.y - lo);
}

struct CutTable { int64_t cuts[RGNN_MAX_WORLD + 1]; int world; };

__global__ void halo_owner_kernel(const uint32_t* __restrict__ halo, int n_halo, const __grid_constant__ CutTable c,
                                  int32_t* __restrict__ g_out, int32_t* __restrict__ owner, int32_t* __restrict__ row) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_halo) return;
  const int64_t g = (int64_t)halo[i];
  int o = 0;
  while (o + 1 < c.world && g >= c.cuts[o + 1]) ++o;
  g_out[i] = (int32_t)g;
  owner[i] = o;
  row[i] = (int32_t)(g - c.cuts[o]);
}

// ---- the exchange -------------------------------------------------------------------------------------------
struct HaloPullParams {
  int rank, world, n_own, n_halo, d;
  const int32_t* owner;
  const int32_t* row;
  const float* peer[RGNN_MAX_WORLD];   // every rank's state buffer (this rank's own at [rank]), mapped here
  float* mine;
  uint32_t* peer_flags[RGNN_MAX_WORLD];   // rank p's flag array [world]; entry [q] is written by rank q
  uint32_t* epoch;
  uint32_t* ticket;
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Peer rows change between exchanges and L1 is not coherent with remote writes: read them with .cg loads (no L1 allocation;
// the lines come from the owner's L2 over NVLink).  NOT ld.volatile: volatile accesses are not coalesced, and 16-byte
// requests over NVLink gave 300 GB/s per rank on 8 GPUs (gpurun_out/r02_bench_d_n8.json) where 128-byte requests do better.
// Ordering: the rows are only read after this CTA's acquire of the owners' flags + __syncthreads().
__device__ __forceinline__ float4 ld_peer4(const float* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

constexpr int HALO_THREADS = 512;
constexpr int HALO_ROWS_IN_FLIGHT = 8;

// The cross-rank barrier of one exchange, run by every CTA: (1) learn the epoch e of this exchange; (2) CTA 0 tells every
// peer "my rows of this buffer are final" (release: the work that wrote them ran earlier on this stream); (3) wait until
// every peer has said the same (acquire).  Returns e.
__device__ __forceinline__ uint32_t exchange_barrier(uint32_t* const* peer_flags, int rank, int world, const uint32_t* epoch) {
  __shared__ uint32_t s_epoch;
  const int tid = threadIdx.x;
  if (tid == 0) s_epoch = *reinterpret_cast<const volatile uint32_t*>(epoch) + 1u;
  __syncthreads();
  const uint32_t e = s_epoch;
  if (blockIdx.x == 0 && tid < world) {
    __threadfence_system();
    st_release_sys(peer_flags[tid] + rank, e);
  }
  if (tid < world) {
    const uint32_t* flag = peer_flags[rank] + tid;
    const unsigned long long t0 = global_ns();
    while ((int32_t)(ld_acquire_sys(flag) - e) < 0) {
      if (global_ns() - t0 > 10000000000ull) __trap();   // 10 s: a peer died -- fault instead of hanging the GPU
    }
  }
  __syncthreads();
  return e;
}

// The last CTA of an exchange to finish publishes its epoch (the next exchange's barrier waits for e + 1).
__device__ __forceinline__ void exchange_done(uint32_t* ticket, uint32_t* epoch, uint32_t e) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned done = atomicAdd(ticket, 1u);
    if (done == gridDim.x - 1) {
      *reinterpret_cast<volatile uint32_t*>(ticket) = 0u;
      *reinterpret_cast<volatile uint32_t*>(epoch) = e;
      __threadfence();
    }
  }
}

// Every CTA: the barrier ("every rank's owned rows of this buffer are final"), then the pull: one warp per halo row, 8 rows
// in flight per warp, 16 bytes per lane per load.  Safe reuse of the two state buffers: a rank overwrites buffer b again only
// after passing the barrier of a LATER exchange, which every peer enters only after its pull from b has completed.
__global__ void __launch_bounds__(HALO_THREADS) halo_pull_kernel(const __grid_constant__ HaloPullParams p) {
  const int tid = threadIdx.x;
  const uint32_t e = exchange_barrier(p.peer_flags, p.rank, p.world, p.epoch);

  const int lane = tid & 31;
  const int warps = (HALO_THREADS / 32) * gridDim.x;
  const int gw = blockIdx.x * (HALO_THREADS / 32) + (tid >> 5);
  const int d = p.d;
  for (int i0 = gw * HALO_ROWS_IN_FLIGHT; i0 < p.n_halo; i0 += warps * HALO_ROWS_IN_FLIGHT) {
    const float* src[HALO_ROWS_IN_FLIGHT];
#pragma unroll
    for (int u = 0; u < HALO_ROWS_IN_FLIGHT; ++u) {
      const int i = i0 + u;
      src[u] = (i < p.n_halo) ? p.peer[__ldg(p.owner + i)] + (size_t)__ldg(p.row + i) * d : nullptr;
    }
    for (int c = lane * 4; c < d; c += 128) {
      float4 v[HALO_ROWS_IN_FLIGHT];
#pragma unroll
      for (int u = 0; u < HALO_ROWS_IN_FLIGHT; ++u)
        if (src[u] != nullptr) v[u] = ld_peer4(src[u] + c);
#pragma unroll
      for (int u = 0; u < HALO_ROWS_IN_FLIGHT; ++u)
        if (src[u] != nullptr) *reinterpret_cast<float4*>(p.mine + (size_t)(p.n_own + i0 + u) * d + c) = v[u];
    }
  }
  exchange_done(p.ticket, p.epoch, e);
}

// ---- the transposed exchange (training) ------------------------------------------------------------------------
struct HaloGradParams {
  int rank, world, n_own, d;
  const int32_t* rev_off;
  const int32_t* rev_peer;
  const int32_t* rev_row;
  const float* peer[RGNN_MAX_WORLD];       // every rank's gradient buffer of this exchange, mapped here
  const float* local;                      // this rank's [n_local, d] gradient (rows [0, n_own) are read)
  float* out;                              // [n_own, d]
  uint32_t* peer_flags[RGNN_MAX_WORLD];    // the GRADIENT flag arrays: never satisfied by a forward exchange
  uint32_t* epoch;
  uint32_t* ticket;
};

// The transpose of halo_pull_kernel.  Every rank has copied the gradients of its halo rows into its gradient buffer (earlier
// on this stream); after the barrier every owner sums, per owned row r, g_local[r] and then the consumers' rows in ascending
// peer rank (the reverse index is sorted that way), one warp per row, 8 rows per warp.  A row without consumers is copied.
// Buffer reuse follows the forward argument: consecutive backward exchanges alternate the two gradient buffers.
__global__ void __launch_bounds__(HALO_THREADS) halo_grad_pull_kernel(const __grid_constant__ HaloGradParams p) {
  const int tid = threadIdx.x;
  const uint32_t e = exchange_barrier(p.peer_flags, p.rank, p.world, p.epoch);

  const int lane = tid & 31;
  const int warps = (HALO_THREADS / 32) * gridDim.x;
  const int gw = blockIdx.x * (HALO_THREADS / 32) + (tid >> 5);
  const int d = p.d;
  for (int r0 = gw * HALO_ROWS_IN_FLIGHT; r0 < p.n_own; r0 += warps * HALO_ROWS_IN_FLIGHT) {
    int beg[HALO_ROWS_IN_FLIGHT], end[HALO_ROWS_IN_FLIGHT];
#pragma unroll
    for (int u = 0; u < HALO_ROWS_IN_FLIGHT; ++u) {
      const int r = r0 + u;
      beg[u] = r < p.n_own ? __ldg(p.rev_off + r) : 0;
      end[u] = r < p.n_own ? __ldg(p.rev_off + r + 1) : 0;
    }
    for (int c = lane * 4; c < d; c += 128) {
#pragma unroll
      for (int u = 0; u < HALO_ROWS_IN_FLIGHT; ++u) {
        const int r = r0 + u;
        if (r >= p.n_own) continue;
        float4 acc = *reinterpret_cast<const float4*>(p.local + (size_t)r * d + c);
        for (int j = beg[u]; j < end[u]; ++j) {
          const float4 v = ld_peer4(p.peer[__ldg(p.rev_peer + j)] + (size_t)__ldg(p.rev_row + j) * d + c);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        *reinterpret_cast<float4*>(p.out + (size_t)r * d + c) = acc;
      }
    }
  }
  exchange_done(p.ticket, p.epoch, e);
}

// ---- the reverse index ------------------------------------------------------------------------------------------
// A published halo list (rgnn_halo_plan_attach_grad): int32 [0] = n_halo, [1..3] = 0, [4, 4 + n_halo) = owner,
// [4 + n_halo, 4 + 2 n_halo) = row inside the owner's buffer.
constexpr int HALO_LIST_HEADER = 4;
constexpr uint64_t REV_SENTINEL = ~0ull;

struct PeerListTable {
  const int32_t* list[RGNN_MAX_WORLD];
  int32_t n[RGNN_MAX_WORLD];        // n_halo of every peer (0 for this rank)
  int32_t off[RGNN_MAX_WORLD];      // first key of peer q
  int32_t n_own[RGNN_MAX_WORLD];    // owned rows of every peer: its halo row i sits at row n_own + i of its buffer
};

__global__ void halo_list_lengths_kernel(const __grid_constant__ PeerListTable t, int world, int rank, int32_t* __restrict__ out) {
  const int q = threadIdx.x;
  if (q < world) out[q] = q == rank ? 0 : t.list[q][0];
}

// key of every entry of every peer's list: (owned row * world + peer) when this rank owns it, else the sentinel; value = the
// row of the peer's gradient buffer.  grid = (ceil(max n / 256), world)
__global__ void halo_rev_keys_kernel(const __grid_constant__ PeerListTable t, int world, int rank, int n_own,
                                     uint64_t* __restrict__ keys, int32_t* __restrict__ vals, int* __restrict__ counters) {
  const int q = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.n[q]) return;
  const int32_t owner = t.list[q][HALO_LIST_HEADER + i];
  const int32_t row = t.list[q][HALO_LIST_HEADER + t.n[q] + i];
  uint64_t key = REV_SENTINEL;
  if (owner == rank) {
    if (row >= 0 && row < n_own) {
      key = (uint64_t)row * (uint64_t)world + (uint64_t)q;
      atomicAdd(counters, 1);
    } else {
      atomicExch(counters + 1, 1);
    }
  }
  keys[t.off[q] + i] = key;
  vals[t.off[q] + i] = t.n_own[q] + i;
}

__device__ __forceinline__ int lower_bound_u64(const uint64_t* a, int n, uint64_t x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// sorted keys (the first n_rev are real) -> CSR offsets over the owned rows + (peer, row) per entry
__global__ void halo_rev_finalize_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, int n_rev,
                                         int n_own, int world, int32_t* __restrict__ off, int32_t* __restrict__ peer,
                                         int32_t* __restrict__ row) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n_own) off[i] = lower_bound_u64(keys, n_rev, (uint64_t)i * (uint64_t)world);
  if (i < n_rev) {
    peer[i] = (int32_t)(keys[i] % (uint64_t)world);
    row[i] = vals[i];
  }
}

}  // namespace
}  // namespace rgnn

using namespace rgnn;

extern "C" int rgnn_halo_plan_destroy(rgnn_halo_plan_t* hp) {
  if (hp == nullptr) return RGNN_OK;
  if (hp->ev_fork != nullptr) cudaEventDestroy(hp->ev_fork);
  if (hp->ev_done != nullptr) cudaEventDestroy(hp->ev_done);
  if (hp->side != nullptr) cudaStreamDestroy(hp->side);
  if (hp->graph != nullptr) rgnn_plan_destroy(hp->graph);
  if (hp->rev_block != nullptr) cudaFreeAsync(hp->rev_block, hp->stream);
  if (hp->block != nullptr) cudaFreeAsync(hp->block, hp->stream);
  delete hp;
  return RGNN_OK;
}

extern "C" int rgnn_halo_plan_create(rgnn_halo_plan_t** out, int32_t rank, int32_t world, const int64_t* cuts,
                                     int32_t num_edge_types, const int32_t* const* adjacency_lists, const int64_t* num_edges,
                                     void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(out != nullptr, "halo_plan_create: out is NULL");
  *out = nullptr;
  RGNN_REQUIRE(world >= 1 && world <= RGNN_MAX_WORLD && rank >= 0 && rank < world, "halo_plan_create: rank %d / world %d invalid (max %d)", rank, world, RGNN_MAX_WORLD);
  RGNN_REQUIRE(cuts != nullptr && adjacency_lists != nullptr && num_edges != nullptr, "halo_plan_create: NULL argument");
  RGNN_REQUIRE(num_edge_types >= 1 && num_edge_types <= RGNN_MAX_EDGE_TYPES, "halo_plan_create: num_edge_types %d outside [1, %d]", num_edge_types, RGNN_MAX_EDGE_TYPES);
  RGNN_REQUIRE(cuts[0] == 0, "halo_plan_create: cuts[0] must be 0");
  for (int r = 0; r < world; ++r) RGNN_REQUIRE(cuts[r + 1] >= cuts[r], "halo_plan_create: cuts must be non-decreasing");
  RGNN_REQUIRE(cuts[world] < (1ll << 31) - 1, "halo_plan_create: more than 2^31 nodes");
  const int L = num_edge_types;
  const int num_global = (int)cuts[world];
  const int lo = (int)cuts[rank], hi = (int)cuts[rank + 1];

  rgnn_halo_plan* hp = new (std::nothrow) rgnn_halo_plan();
  RGNN_REQUIRE(hp != nullptr, "halo_plan_create: out of host memory");
  hp->rank = rank; hp->world = world; hp->lo = lo; hp->n_own = hi - lo; hp->L = L; hp->stream = stream;
  for (int r = 0; r <= world; ++r) hp->cuts[r] = cuts[r];
  cudaGetDevice(&hp->device);
  auto fail = [&](int code) { rgnn_halo_plan_destroy(hp); return code; };
#define HALO_CUDA(expr)                                                                                   \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
      if (scratch) cudaFreeAsync(scratch, stream);                                                         \
      return fail(RGNN_E_CUDA);                                                                            \
    }                                                                                                      \
  } while (0)

  int64_t total_in = 0, max_in = 0;
  for (int l = 0; l < L; ++l) {
    if (num_edges[l] < 0 || (num_edges[l] > 0 && (adjacency_lists[l] == nullptr || (reinterpret_cast<uintptr_t>(adjacency_lists[l]) & 7u)))) {
      set_error("halo_plan_create: adjacency list %d is NULL / misaligned / negative length", l);
      return fail(RGNN_E_INVALID);
    }
    total_in += num_edges[l];
    if (num_edges[l] > max_in) max_in = num_edges[l];
  }
  if (total_in >= (1ll << 31)) { set_error("halo_plan_create: more than 2^31 edges"); return fail(RGNN_E_UNSUPPORTED); }

  // ---- scratch: kept edges (upper bound: all input edges), keys x2, unique list, counters, CUB temp ----
  char* scratch = nullptr;
  const size_t Mz = (size_t)(total_in > 0 ? total_in : 1);
  const size_t kept_bytes = align_up(Mz * sizeof(int2), 256);
  const size_t key_bytes = align_up(Mz * sizeof(uint32_t), 256);
  size_t cub_sel = 0, cub_sort = 0, cub_unique = 0;
  {
    OwnedTarget op{lo, hi};
    HALO_CUDA(cub::DeviceSelect::If(nullptr, cub_sel, (const int2*)nullptr, (int2*)nullptr, (int*)nullptr, (int)(max_in > 0 ? max_in : 1), op, stream));
    HALO_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, cub_sort, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)Mz, 0, 32, stream));
    HALO_CUDA(cub::DeviceSelect::Unique(nullptr, cub_unique, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int*)nullptr, (int)Mz, stream));
  }
  size_t cub_bytes = cub_sel > cub_sort ? cub_sel : cub_sort;
  if (cub_unique > cub_bytes) cub_bytes = cub_unique;
  cub_bytes = align_up(cub_bytes, 256);
  const size_t counters_bytes = 256 * sizeof(int);   // [0..L) kept counts, [L] num_unique, [L+1] n_halo, [L+2] error flag
  HALO_CUDA(cudaMallocAsync(&scratch, kept_bytes + 3 * key_bytes + counters_bytes + cub_bytes, stream));
  int2* kept = reinterpret_cast<int2*>(scratch);
  uint32_t* keys0 = reinterpret_cast<uint32_t*>(scratch + kept_bytes);
  uint32_t* keys1 = reinterpret_cast<uint32_t*>(scratch + kept_bytes + key_bytes);
  uint32_t* uniq = reinterpret_cast<uint32_t*>(scratch + kept_bytes + 2 * key_bytes);
  int* counters = reinterpret_cast<int*>(scratch + kept_bytes + 3 * key_bytes);
  void* cub_tmp = scratch + kept_bytes + 3 * key_bytes + counters_bytes;
  HALO_CUDA(cudaMemsetAsync(counters, 0, counters_bytes, stream));

  // (1) keep the edges whose target this rank owns, per type, order preserved
  {
    int64_t in_off = 0;
    for (int l = 0; l < L; ++l) {
      if (num_edges[l] > 0) {
        OwnedTarget op{lo, hi};
        size_t tmp = cub_bytes;
        HALO_CUDA(cub::DeviceSelect::If(cub_tmp, tmp, reinterpret_cast<const int2*>(adjacency_lists[l]), kept + in_off, counters + l,
                                        (int)num_edges[l], op, stream));
        count_launch();
      }
      in_off += num_edges[l];
    }
  }
  int host_counts[RGNN_MAX_EDGE_TYPES + 3] = {0};
  HALO_CUDA(cudaMemcpyAsync(host_counts, counters, sizeof(int) * L, cudaMemcpyDeviceToHost, stream));
  HALO_CUDA(cudaStreamSynchronize(stream));
  KeptTable kt;
  int64_t M = 0;
  int32_t maxE = 0;
  {
    int64_t in_off = 0;
    for (int l = 0; l < L; ++l) {
      kt.adj[l] = kept + in_off;
      kt.count[l] = host_counts[l];
      kt.off[l] = (int32_t)M;
      hp->num_edges[l] = host_counts[l];
      M += host_counts[l];
      if (host_counts[l] > maxE) maxE = host_counts[l];
      in_off += num_edges[l];
    }
  }

  // (2) distinct remote sources = the halo list (sorted by global id)
  int n_halo = 0;
  if (M > 0) {
    halo_keys_kernel<<<dim3((maxE + 255) / 256, L), 256, 0, stream>>>(kt, lo, hi, num_global, keys0, counters + L + 2);
    HALO_CUDA(cudaGetLastError());
    count_launch();
    size_t tmp = cub_bytes;
    HALO_CUDA(cub::DeviceRadixSort::SortKeys(cub_tmp, tmp, keys0, keys1, (int)M, 0, 32, stream));
    tmp = cub_bytes;
    HALO_CUDA(cub::DeviceSelect::Unique(cub_tmp, tmp, keys1, uniq, counters + L, (int)M, stream));
    halo_count_kernel<<<1, 1, 0, stream>>>(uniq, counters + L, counters + L + 1);
    HALO_CUDA(cudaGetLastError());
    count_launch(3);
    HALO_CUDA(cudaMemcpyAsync(host_counts + L, counters + L, sizeof(int) * 3, cudaMemcpyDeviceToHost, stream));
    HALO_CUDA(cudaStreamSynchronize(stream));
    n_halo = host_counts[L + 1];
    if (host_counts[L + 2] != 0) {
      cudaFreeAsync(scratch, stream);
      set_error("halo_plan_create: an adjacency list holds a node index outside [0, %d)", num_global);
      return fail(RGNN_E_INVALID);
    }
  }
  hp->n_halo = n_halo;
  hp->n_local = hp->n_own + n_halo;

  // (3) the plan's own arrays: local adjacency lists, halo lists, exchange counters
  {
    const size_t adj_bytes = align_up((size_t)(M > 0 ? M : 1) * sizeof(int2), 256);
    const size_t h_bytes = align_up((size_t)(n_halo > 0 ? n_halo : 1) * sizeof(int32_t), 256);
    HALO_CUDA(cudaMallocAsync(&hp->block, adj_bytes + 3 * h_bytes + 256, stream));
    char* b = static_cast<char*>(hp->block);
    for (int l = 0; l < L; ++l) hp->local_adj[l] = reinterpret_cast<int32_t*>(b) + 2 * (size_t)kt.off[l];
    hp->halo_global = reinterpret_cast<int32_t*>(b + adj_bytes);
    hp->halo_owner = reinterpret_cast<int32_t*>(b + adj_bytes + h_bytes);
    hp->halo_row = reinterpret_cast<int32_t*>(b + adj_bytes + 2 * h_bytes);
    hp->epoch = reinterpret_cast<uint32_t*>(b + adj_bytes + 3 * h_bytes);
    hp->ticket = hp->epoch + 1;
    hp->grad_epoch = hp->epoch + 2;
    hp->grad_ticket = hp->epoch + 3;
    HALO_CUDA(cudaMemsetAsync(hp->epoch, 0, 256, stream));
  }
  if (M > 0) {
    LocalTable lt;
    for (int l = 0; l < L; ++l) lt.adj[l] = hp->local_adj[l];
    halo_renumber_kernel<<<dim3((maxE + 255) / 256, L), 256, 0, stream>>>(kt, lt, lo, hi, hp->n_own, uniq, n_halo);
    HALO_CUDA(cudaGetLastError());
    count_launch();
  }
  if (n_halo > 0) {
    CutTable ct;
    ct.world = world;
    for (int r = 0; r <= world; ++r) ct.cuts[r] = cuts[r];
    halo_owner_kernel<<<(n_halo + 255) / 256, 256, 0, stream>>>(uniq, n_halo, ct, hp->halo_global, hp->halo_owner, hp->halo_row);
    HALO_CUDA(cudaGetLastError());
    count_launch();
  }
  HALO_CUDA(cudaFreeAsync(scratch, stream));
  scratch = nullptr;
#undef HALO_CUDA

  // (4) the ordinary plan over local ids, outputs restricted to the owned rows
  {
    const int32_t* ptrs[RGNN_MAX_EDGE_TYPES];
    for (int l = 0; l < L; ++l) ptrs[l] = hp->local_adj[l];
    const int rc = rgnn_plan_create_ex(&hp->graph, hp->n_local, L, ptrs, hp->num_edges, 0, stream);
    if (rc != RGNN_OK) return fail(rc);
    rgnn_plan_set_num_targets(hp->graph, hp->n_own);
  }
  *out = hp;
  return RGNN_OK;
}

extern "C" int32_t rgnn_halo_plan_num_own(const rgnn_halo_plan_t* hp) { return hp ? hp->n_own : -1; }
extern "C" int32_t rgnn_halo_plan_num_halo(const rgnn_halo_plan_t* hp) { return hp ? hp->n_halo : -1; }
extern "C" int64_t rgnn_halo_plan_num_edges(const rgnn_halo_plan_t* hp, int32_t edge_type) {
  return (hp && edge_type >= 0 && edge_type < hp->L) ? hp->num_edges[edge_type] : -1;
}
extern "C" rgnn_plan_t* rgnn_halo_plan_graph(rgnn_halo_plan_t* hp) { return hp ? hp->graph : nullptr; }

extern "C" int rgnn_halo_plan_export(const rgnn_halo_plan_t* hp, int32_t* halo_global, int32_t* halo_owner, int32_t* halo_row,
                                     int32_t* const* local_adjacency_lists, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(hp != nullptr, "halo_plan_export: plan is NULL");
  const size_t hb = sizeof(int32_t) * (size_t)hp->n_halo;
  if (halo_global && hb) RGNN_CHECK_CUDA(cudaMemcpyAsync(halo_global, hp->halo_global, hb, cudaMemcpyDeviceToDevice, stream));
  if (halo_owner && hb) RGNN_CHECK_CUDA(cudaMemcpyAsync(halo_owner, hp->halo_owner, hb, cudaMemcpyDeviceToDevice, stream));
  if (halo_row && hb) RGNN_CHECK_CUDA(cudaMemcpyAsync(halo_row, hp->halo_row, hb, cudaMemcpyDeviceToDevice, stream));
  if (local_adjacency_lists != nullptr)
    for (int l = 0; l < hp->L; ++l)
      if (local_adjacency_lists[l] != nullptr && hp->num_edges[l] > 0)
        RGNN_CHECK_CUDA(cudaMemcpyAsync(local_adjacency_lists[l], hp->local_adj[l], sizeof(int32_t) * 2 * (size_t)hp->num_edges[l],
                                        cudaMemcpyDeviceToDevice, stream));
  return RGNN_OK;
}

extern "C" int rgnn_halo_plan_attach(rgnn_halo_plan_t* hp, void* const* peer_states0, void* const* peer_states1,
                                     void* const* peer_flags) {
  RGNN_REQUIRE(hp != nullptr && peer_states0 != nullptr && peer_states1 != nullptr && peer_flags != nullptr, "halo_plan_attach: NULL argument");
  for (int r = 0; r < hp->world; ++r) {
    RGNN_REQUIRE(peer_states0[r] != nullptr && peer_states1[r] != nullptr && peer_flags[r] != nullptr, "halo_plan_attach: pointer of rank %d is NULL", r);
    RGNN_REQUIRE(aligned16(peer_states0[r]) && aligned16(peer_states1[r]), "halo_plan_attach: state buffers must be 16-byte aligned");
    hp->peer_state[0][r] = static_cast<float*>(peer_states0[r]);
    hp->peer_state[1][r] = static_cast<float*>(peer_states1[r]);
    hp->peer_flags[r] = static_cast<uint32_t*>(peer_flags[r]);
  }
  hp->attached = true;
  return RGNN_OK;
}

static int halo_exchange_on(rgnn_halo_plan_t* hp, int buffer, int32_t d, cudaStream_t stream);

extern "C" int rgnn_halo_exchange(rgnn_halo_plan_t* hp, int buffer, int32_t d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // two exchange kernels of one plan must never run concurrently (they share the epoch / ticket counters): an overlapped
  // exchange that no layer forward has joined yet is joined here first
  if (hp != nullptr && hp->graph != nullptr) RGNN_PROPAGATE(plan_wait_sources(hp->graph, stream));
  return halo_exchange_on(hp, buffer, d, stream);
}

// The same exchange, off the caller's critical path: forked onto the plan's side stream (after everything enqueued on `stream`
// so far), NOT joined here -- the next layer forward on rgnn_halo_plan_graph() joins it right before its first kernel that reads
// halo rows, so the layer's target-side work (FiLM's gamma / beta GEMM over the owned rows) overlaps the pull over NVLink.
extern "C" int rgnn_halo_exchange_overlapped(rgnn_halo_plan_t* hp, int buffer, int32_t d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(hp != nullptr && hp->attached, "halo_exchange_overlapped: plan is NULL / peer memory not attached");
  if (hp->side == nullptr) {
    RGNN_CHECK_CUDA(cudaStreamCreateWithFlags(&hp->side, cudaStreamNonBlocking));
    RGNN_CHECK_CUDA(cudaEventCreateWithFlags(&hp->ev_fork, cudaEventDisableTiming));
    RGNN_CHECK_CUDA(cudaEventCreateWithFlags(&hp->ev_done, cudaEventDisableTiming));
  }
  RGNN_PROPAGATE(plan_wait_sources(hp->graph, stream));        // an unconsumed earlier exchange is joined first
  RGNN_CHECK_CUDA(cudaEventRecord(hp->ev_fork, stream));
  RGNN_CHECK_CUDA(cudaStreamWaitEvent(hp->side, hp->ev_fork, 0));
  RGNN_PROPAGATE(halo_exchange_on(hp, buffer, d, hp->side));
  RGNN_CHECK_CUDA(cudaEventRecord(hp->ev_done, hp->side));
  hp->graph->source_ready = hp->ev_done;
  return RGNN_OK;
}

static int halo_exchange_on(rgnn_halo_plan_t* hp, int buffer, int32_t d, cudaStream_t stream) {
  RGNN_REQUIRE(hp != nullptr, "halo_exchange: plan is NULL");
  RGNN_REQUIRE(hp->attached, "halo_exchange: peer memory not attached (rgnn_halo_plan_attach)");
  RGNN_REQUIRE(buffer == 0 || buffer == 1, "halo_exchange: buffer %d is not 0 or 1", buffer);
  RGNN_REQUIRE(d > 0 && (d % 4) == 0, "halo_exchange: state dim %d must be a positive multiple of 4", d);
  HaloPullParams p;
  p.rank = hp->rank; p.world = hp->world; p.n_own = hp->n_own; p.n_halo = hp->n_halo; p.d = d;
  p.owner = hp->halo_owner; p.row = hp->halo_row;
  for (int r = 0; r < hp->world; ++r) { p.peer[r] = hp->peer_state[buffer][r]; p.peer_flags[r] = hp->peer_flags[r]; }
  p.mine = hp->peer_state[buffer][hp->rank];
  p.epoch = hp->epoch; p.ticket = hp->ticket;
  // enough warps to keep ~150 k 16-byte loads in flight over NVLink, never more CTAs than are co-resident
  const long warps_needed = ((long)hp->n_halo + HALO_ROWS_IN_FLIGHT - 1) / HALO_ROWS_IN_FLIGHT;
  long ctas = (warps_needed + HALO_THREADS / 32 - 1) / (HALO_THREADS / 32);
  if (ctas < 1) ctas = 1;
  if (ctas > 2 * RGNN_WAVE_SMS) ctas = 2 * RGNN_WAVE_SMS;
  halo_pull_kernel<<<(unsigned)ctas, HALO_THREADS, 0, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

// ---- training: the transposed exchange -----------------------------------------------------------------------------
extern "C" int rgnn_halo_plan_attach_grad(rgnn_halo_plan_t* hp, void* const* peer_grads0, void* const* peer_grads1,
                                          void* const* peer_grad_flags, void* const* peer_halo_lists) {
  RGNN_REQUIRE(hp != nullptr && peer_grads0 != nullptr && peer_grads1 != nullptr && peer_grad_flags != nullptr &&
               peer_halo_lists != nullptr, "halo_plan_attach_grad: NULL argument");
  for (int r = 0; r < hp->world; ++r) {
    RGNN_REQUIRE(peer_grads0[r] != nullptr && peer_grads1[r] != nullptr && peer_grad_flags[r] != nullptr &&
                 peer_halo_lists[r] != nullptr, "halo_plan_attach_grad: pointer of rank %d is NULL", r);
    RGNN_REQUIRE(aligned16(peer_grads0[r]) && aligned16(peer_grads1[r]) && aligned16(peer_halo_lists[r]),
                 "halo_plan_attach_grad: gradient buffers and halo lists must be 16-byte aligned");
    RGNN_REQUIRE(peer_grad_flags[r] != static_cast<void*>(hp->peer_flags[r]),
                 "halo_plan_attach_grad: the gradient flags of rank %d are the forward exchange's flags", r);
  }
  // Load both exchange kernels now.  With lazy module loading (CUDA's default) a kernel is loaded at its first launch, and
  // loading can wait for the kernels running on the device -- among them an exchange spinning for a peer that this very
  // host thread has yet to enqueue (virtual ranks).
  cudaFuncAttributes fa;
  RGNN_CHECK_CUDA(cudaFuncGetAttributes(&fa, halo_pull_kernel));
  RGNN_CHECK_CUDA(cudaFuncGetAttributes(&fa, halo_grad_pull_kernel));
  // publish this rank's halo list (read by the peers' rgnn_halo_plan_build_reverse); finished when this call returns
  int32_t* mine = static_cast<int32_t*>(peer_halo_lists[hp->rank]);
  const int32_t header[HALO_LIST_HEADER] = {hp->n_halo, 0, 0, 0};
  const size_t hb = sizeof(int32_t) * (size_t)hp->n_halo;
  cudaStream_t s = nullptr;
  RGNN_CHECK_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  cudaError_t e = cudaMemcpyAsync(mine, header, sizeof(header), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess && hb) e = cudaMemcpyAsync(mine + HALO_LIST_HEADER, hp->halo_owner, hb, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess && hb) e = cudaMemcpyAsync(mine + HALO_LIST_HEADER + hp->n_halo, hp->halo_row, hb, cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaStreamDestroy(s);
  if (e != cudaSuccess) {
    set_error("halo_plan_attach_grad: %s (%s)", cudaGetErrorName(e), cudaGetErrorString(e));
    return RGNN_E_CUDA;
  }
  for (int r = 0; r < hp->world; ++r) {
    hp->peer_grad[0][r] = static_cast<float*>(peer_grads0[r]);
    hp->peer_grad[1][r] = static_cast<float*>(peer_grads1[r]);
    hp->peer_grad_flags[r] = static_cast<uint32_t*>(peer_grad_flags[r]);
    hp->peer_lists[r] = static_cast<const int32_t*>(peer_halo_lists[r]);
  }
  hp->grad_attached = true;
  hp->n_rev = -1;                                   // the peers' lists may have changed: build the index again
  return RGNN_OK;
}

static int end_bit_above(uint64_t n) {             // smallest b with 2^b > n
  int b = 1;
  while (b < 64 && (1ull << b) <= n) ++b;
  return b;
}

extern "C" int rgnn_halo_plan_build_reverse(rgnn_halo_plan_t* hp, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(hp != nullptr, "halo_plan_build_reverse: plan is NULL");
  RGNN_REQUIRE(hp->grad_attached, "halo_plan_build_reverse: gradient memory not attached (rgnn_halo_plan_attach_grad)");
  {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    RGNN_CHECK_CUDA(cudaStreamIsCapturing(stream, &cap));
    RGNN_REQUIRE(cap == cudaStreamCaptureStatusNone,
                 "halo_plan_build_reverse: synchronises the stream, which is capturing a CUDA graph (build the reverse "
                 "index eagerly, before capturing)");
  }
  const int world = hp->world, rank = hp->rank, n_own = hp->n_own;
  PeerListTable t;
  for (int q = 0; q < RGNN_MAX_WORLD; ++q) {
    t.list[q] = q < world ? hp->peer_lists[q] : nullptr;
    t.n[q] = 0;
    t.off[q] = 0;
    t.n_own[q] = q < world ? (int32_t)(hp->cuts[q + 1] - hp->cuts[q]) : 0;
  }
  int32_t* small = nullptr;                         // [0, world) list lengths, [32] entries owned here, [33] error flag
  char* scratch = nullptr;
  void* block = nullptr;
  auto cleanup = [&]() {
    if (block != nullptr) cudaFreeAsync(block, stream);
    if (scratch != nullptr) cudaFreeAsync(scratch, stream);
    if (small != nullptr) cudaFreeAsync(small, stream);
    cudaStreamSynchronize(stream);
  };
#define REV_CUDA(expr)                                                                                    \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
      cleanup();                                                                                           \
      return RGNN_E_CUDA;                                                                                  \
    }                                                                                                      \
  } while (0)

  RGNN_CHECK_CUDA(cudaMallocAsync(&small, 256, stream));
  REV_CUDA(cudaMemsetAsync(small, 0, 256, stream));
  halo_list_lengths_kernel<<<1, 32, 0, stream>>>(t, world, rank, small);
  REV_CUDA(cudaGetLastError());
  count_launch();
  int32_t len[RGNN_MAX_WORLD] = {0};
  REV_CUDA(cudaMemcpyAsync(len, small, sizeof(int32_t) * world, cudaMemcpyDeviceToHost, stream));
  REV_CUDA(cudaStreamSynchronize(stream));
  int64_t total = 0;
  int32_t max_n = 0;
  for (int q = 0; q < world; ++q) {
    if (len[q] < 0 || len[q] > hp->cuts[world]) {
      set_error("halo_plan_build_reverse: the published halo list of rank %d claims %d entries", q, len[q]);
      cleanup();
      return RGNN_E_INVALID;
    }
    t.n[q] = len[q];
    t.off[q] = (int32_t)total;
    total += len[q];
    if (len[q] > max_n) max_n = len[q];
  }
  if (total >= (1ll << 31)) {
    set_error("halo_plan_build_reverse: more than 2^31 halo entries over the peers");
    cleanup();
    return RGNN_E_UNSUPPORTED;
  }

  // (owned row, peer) keys of the entries this rank owns, radix-sorted; the rest sort to the end
  int n_rev = 0;
  const uint64_t* keys = nullptr;
  const int32_t* vals = nullptr;
  if (total > 0) {
    const int end_bit = end_bit_above((uint64_t)n_own * (uint64_t)world);
    size_t cub_bytes = 0;
    {
      cub::DoubleBuffer<uint64_t> dk(nullptr, nullptr);
      cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
      REV_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, dk, dv, (int)total, 0, end_bit, stream));
    }
    const size_t kb = align_up(sizeof(uint64_t) * (size_t)total, 256), vb = align_up(sizeof(int32_t) * (size_t)total, 256);
    REV_CUDA(cudaMallocAsync(&scratch, 2 * kb + 2 * vb + align_up(cub_bytes, 256), stream));
    uint64_t* k0 = reinterpret_cast<uint64_t*>(scratch);
    uint64_t* k1 = reinterpret_cast<uint64_t*>(scratch + kb);
    int32_t* v0 = reinterpret_cast<int32_t*>(scratch + 2 * kb);
    int32_t* v1 = reinterpret_cast<int32_t*>(scratch + 2 * kb + vb);
    halo_rev_keys_kernel<<<dim3((max_n + 255) / 256, world), 256, 0, stream>>>(t, world, rank, n_own, k0, v0, small + 32);
    REV_CUDA(cudaGetLastError());
    count_launch();
    cub::DoubleBuffer<uint64_t> dk(k0, k1);
    cub::DoubleBuffer<int32_t> dv(v0, v1);
    REV_CUDA(cub::DeviceRadixSort::SortPairs(scratch + 2 * kb + 2 * vb, cub_bytes, dk, dv, (int)total, 0, end_bit, stream));
    count_launch();
    int32_t counts[2] = {0, 0};
    REV_CUDA(cudaMemcpyAsync(counts, small + 32, sizeof(counts), cudaMemcpyDeviceToHost, stream));
    REV_CUDA(cudaStreamSynchronize(stream));
    if (counts[1] != 0) {
      set_error("halo_plan_build_reverse: a peer's halo list names a row of rank %d outside [0, %d)", rank, n_own);
      cleanup();
      return RGNN_E_INVALID;
    }
    n_rev = counts[0];
    keys = dk.Current();
    vals = dv.Current();
  }

  // the index: CSR offsets over the owned rows, (peer, row) per entry
  const size_t off_bytes = align_up(sizeof(int32_t) * ((size_t)n_own + 1), 256);
  const size_t e_bytes = align_up(sizeof(int32_t) * (size_t)(n_rev > 0 ? n_rev : 1), 256);
  REV_CUDA(cudaMallocAsync(&block, off_bytes + 2 * e_bytes, stream));
  int32_t* off = static_cast<int32_t*>(block);
  int32_t* peer = reinterpret_cast<int32_t*>(static_cast<char*>(block) + off_bytes);
  int32_t* row = reinterpret_cast<int32_t*>(static_cast<char*>(block) + off_bytes + e_bytes);
  if (total > 0) {
    const int n = n_rev > n_own + 1 ? n_rev : n_own + 1;
    halo_rev_finalize_kernel<<<(n + 255) / 256, 256, 0, stream>>>(keys, vals, n_rev, n_own, world, off, peer, row);
    REV_CUDA(cudaGetLastError());
    count_launch();
  } else {
    REV_CUDA(cudaMemsetAsync(off, 0, sizeof(int32_t) * ((size_t)n_own + 1), stream));
  }
  if (hp->rev_block != nullptr) cudaFreeAsync(hp->rev_block, stream);
  hp->rev_block = block;
  hp->rev_off = off;
  hp->rev_peer = peer;
  hp->rev_row = row;
  hp->n_rev = n_rev;
  block = nullptr;
  cleanup();
#undef REV_CUDA
  RGNN_CHECK_CUDA(cudaGetLastError());
  return RGNN_OK;
}

extern "C" int64_t rgnn_halo_plan_num_reverse(const rgnn_halo_plan_t* hp) { return hp ? hp->n_rev : -1; }

extern "C" int rgnn_halo_plan_export_reverse(const rgnn_halo_plan_t* hp, int32_t* offsets, int32_t* peer, int32_t* row,
                                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(hp != nullptr, "halo_plan_export_reverse: plan is NULL");
  RGNN_REQUIRE(hp->n_rev >= 0, "halo_plan_export_reverse: reverse index not built (rgnn_halo_plan_build_reverse)");
  const size_t eb = sizeof(int32_t) * (size_t)hp->n_rev;
  if (offsets) RGNN_CHECK_CUDA(cudaMemcpyAsync(offsets, hp->rev_off, sizeof(int32_t) * ((size_t)hp->n_own + 1), cudaMemcpyDeviceToDevice, stream));
  if (peer && eb) RGNN_CHECK_CUDA(cudaMemcpyAsync(peer, hp->rev_peer, eb, cudaMemcpyDeviceToDevice, stream));
  if (row && eb) RGNN_CHECK_CUDA(cudaMemcpyAsync(row, hp->rev_row, eb, cudaMemcpyDeviceToDevice, stream));
  return RGNN_OK;
}

extern "C" int rgnn_halo_exchange_backward(rgnn_halo_plan_t* hp, int buffer, int32_t d, const float* grad_local,
                                           float* grad_own, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(hp != nullptr, "halo_exchange_backward: plan is NULL");
  RGNN_REQUIRE(hp->grad_attached, "halo_exchange_backward: gradient memory not attached (rgnn_halo_plan_attach_grad)");
  RGNN_REQUIRE(hp->n_rev >= 0, "halo_exchange_backward: reverse index not built (rgnn_halo_plan_build_reverse)");
  RGNN_REQUIRE(buffer == 0 || buffer == 1, "halo_exchange_backward: buffer %d is not 0 or 1", buffer);
  RGNN_REQUIRE(d > 0 && (d % 4) == 0, "halo_exchange_backward: gradient dim %d must be a positive multiple of 4", d);
  RGNN_REQUIRE((grad_local != nullptr || hp->n_local == 0) && (grad_own != nullptr || hp->n_own == 0),
               "halo_exchange_backward: gradient pointer is NULL");
  RGNN_REQUIRE(aligned16(grad_local) && aligned16(grad_own), "halo_exchange_backward: gradients must be 16-byte aligned");
  // this rank's halo-row gradients -> its peer-visible buffer (skipped when the caller computed them there)
  float* mine = hp->peer_grad[buffer][hp->rank];
  const size_t halo_off = (size_t)hp->n_own * d;
  if (hp->n_halo > 0 && grad_local + halo_off != mine + halo_off)
    RGNN_CHECK_CUDA(cudaMemcpyAsync(mine + halo_off, grad_local + halo_off, sizeof(float) * (size_t)hp->n_halo * d,
                                    cudaMemcpyDeviceToDevice, stream));
  HaloGradParams p;
  p.rank = hp->rank; p.world = hp->world; p.n_own = hp->n_own; p.d = d;
  p.rev_off = hp->rev_off; p.rev_peer = hp->rev_peer; p.rev_row = hp->rev_row;
  for (int r = 0; r < hp->world; ++r) { p.peer[r] = hp->peer_grad[buffer][r]; p.peer_flags[r] = hp->peer_grad_flags[r]; }
  p.local = grad_local; p.out = grad_own;
  p.epoch = hp->grad_epoch; p.ticket = hp->grad_ticket;
  // the forward's sizing, over the owned rows; never more CTAs than are co-resident
  const long warps_needed = ((long)hp->n_own + HALO_ROWS_IN_FLIGHT - 1) / HALO_ROWS_IN_FLIGHT;
  long ctas = (warps_needed + HALO_THREADS / 32 - 1) / (HALO_THREADS / 32);
  if (ctas < 1) ctas = 1;
  if (ctas > 2 * RGNN_WAVE_SMS) ctas = 2 * RGNN_WAVE_SMS;
  halo_grad_pull_kernel<<<(unsigned)ctas, HALO_THREADS, 0, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

// ---- peer memory: device allocations that other processes on this node can map (CUDA IPC) ---------------------
extern "C" int rgnn_peer_alloc(void** ptr, size_t bytes, void* handle_out) {
  RGNN_REQUIRE(ptr != nullptr && handle_out != nullptr && bytes > 0, "peer_alloc: bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == RGNN_PEER_HANDLE_BYTES, "IPC handle size");
  void* p = nullptr;
  RGNN_CHECK_CUDA(cudaMalloc(&p, bytes));
  cudaError_t e = cudaMemset(p, 0, bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    set_error("peer_alloc: %s (%s)", cudaGetErrorName(e), cudaGetErrorString(e));
    return RGNN_E_CUDA;
  }
  memcpy(handle_out, &h, sizeof(h));
  *ptr = p;
  return RGNN_OK;
}
extern "C" int rgnn_peer_open(const void* handle, void** ptr) {
  RGNN_REQUIRE(handle != nullptr && ptr != nullptr, "peer_open: bad argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  RGNN_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return RGNN_OK;
}
extern "C" int rgnn_peer_close(void* ptr) {
  if (ptr != nullptr) RGNN_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
  return RGNN_OK;
}
extern "C" int rgnn_peer_free(void* ptr) {
  if (ptr != nullptr) RGNN_CHECK_CUDA(cudaFree(ptr));
  return RGNN_OK;
}
