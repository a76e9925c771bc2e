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

// Every CTA: (1) learn the epoch e of this exchange; (2) CTA 0 tells every peer "my owned rows of this buffer are final"
// (release: the layer kernel that wrote them ran earlier on this stream); (3) wait until every peer has said the same
// (acquire); (4) pull: one warp per halo row, 8 rows in flight per warp, 16 bytes per lane per load.  The last CTA to finish
// publishes the new epoch.  Safe reuse of the two state buffers: a rank overwrites buffer b again only after passing the
// barrier of a LATER exchange, which every peer enters only after its pull from b has completed.
__global__ void __launch_bounds__(HALO_THREADS) halo_pull_kernel(const __grid_constant__ HaloPullParams p) {
  __shared__ uint32_t s_epoch;
  const int tid = threadIdx.x;
  if (tid == 0) s_epoch = *reinterpret_cast<volatile uint32_t*>(p.epoch) + 1u;
  __syncthreads();
  const uint32_t e = s_epoch;
  if (blockIdx.x == 0 && tid < p.world) {
    __threadfence_system();
    st_release_sys(p.peer_flags[tid] + p.rank, e);
  }
  if (tid < p.world) {
    const uint32_t* flag = p.peer_flags[p.rank] + tid;
    const unsigned long long t0 = global_ns();
    while ((int32_t)(ld_acquire_sys(flag) - e) < 0) {
      if (global_ns() - t0 > 10000000000ull) __trap();   // 10 s: a peer died -- fault instead of hanging the GPU
    }
  }
  __syncthreads();

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

  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const unsigned done = atomicAdd(p.ticket, 1u);
    if (done == gridDim.x - 1) {
      *reinterpret_cast<volatile uint32_t*>(p.ticket) = 0u;
      *reinterpret_cast<volatile uint32_t*>(p.epoch) = e;
      __threadfence();
    }
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
