// plan.cu -- build the per-batch graph plan on the device.
//
// The reference concatenates the per-type target lists into unsorted segment ids every layer
// (gnns/rgcn.py:76-78) and scatter-adds [M, D] messages with tf.unsorted_segment_* (rgcn.py:110).
// Here the batch's adjacency lists (the task batcher's output, tasks/ppi_task.py:197-256) are
// turned ONCE per batch into a CSR-by-target over all edge types, which every layer / timestep
// reuses: each target's incoming messages become one contiguous, deterministic, atomic-free
// segment.  Sorting uses CUB's stable radix sort (toolkit header library; batch preprocessing,
// not the per-layer hot path -- SURVEY.md 8f row 3).
#include "plan.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <new>
#include <stdlib.h>

namespace rgnn {

namespace {

struct AdjTable {
  const int32_t* adj[RGNN_MAX_EDGE_TYPES];
  int32_t count[RGNN_MAX_EDGE_TYPES];
  int32_t off[RGNN_MAX_EDGE_TYPES];
};

// grid = (ceil(maxE / 256), L)
__global__ void plan_concat_kernel(const __grid_constant__ AdjTable t, int V, int L, int32_t* __restrict__ o_src,
                                   int32_t* __restrict__ o_tgt, uint32_t* __restrict__ keys,
                                   int32_t* __restrict__ vals, int* __restrict__ err) {
  const int l = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.count[l]) return;
  const int2 e = __ldg(reinterpret_cast<const int2*>(t.adj[l]) + i);   // (src, tgt): gnns/rgcn.py:85-86
  const int pos = t.off[l] + i;
  int src = e.x, tgt = e.y;
  if (src < 0 || src >= V || tgt < 0 || tgt >= V) {                    // TF would fail the gather at sess.run
    atomicExch(err, 1);
    src = 0; tgt = 0;
  }
  o_src[pos] = src;
  o_tgt[pos] = tgt;
  keys[pos] = (uint32_t)tgt * (uint32_t)L + (uint32_t)l;
  vals[pos] = pos;
}

__global__ void plan_finalize_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                     const int32_t* __restrict__ o_src, int V, int L, int M,
                                     int32_t* __restrict__ seg_off, int32_t* __restrict__ e_src,
                                     int32_t* __restrict__ e_type, int32_t* __restrict__ e_orig) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M) return;
  const uint32_t k = keys[e];
  const int tgt = (int)(k / (uint32_t)L);
  const int orig = vals[e];
  e_src[e] = o_src[orig];
  e_type[e] = (int)(k % (uint32_t)L);
  e_orig[e] = orig;
  const int prev = (e == 0) ? -1 : (int)(keys[e - 1] / (uint32_t)L);
  for (int v = prev + 1; v <= tgt; ++v) seg_off[v] = e;       // first edge of v (and of empty nodes before it)
  if (e == M - 1)
    for (int v = tgt + 1; v <= V; ++v) seg_off[v] = M;
}

struct TypeOffsets { int32_t off[RGNN_MAX_EDGE_TYPES + 1]; };

// keys for the reverse index: (source * L + type) of every edge in original (type-major) order
__global__ void plan_rev_keys_kernel(const __grid_constant__ TypeOffsets t, int L, const int32_t* __restrict__ o_src,
                                     uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
  const int l = blockIdx.y;
  const int i = t.off[l] + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.off[l + 1]) return;
  keys[i] = (uint32_t)o_src[i] * (uint32_t)L + (uint32_t)l;
  vals[i] = i;
}

__global__ void plan_rev_finalize_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                         const int32_t* __restrict__ o_tgt, int segments, int L, int M,
                                         int32_t* __restrict__ seg_off, int32_t* __restrict__ r_src,
                                         int32_t* __restrict__ r_type) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M) return;
  const int seg = (int)keys[e];
  r_src[e] = o_tgt[vals[e]];
  r_type[e] = seg % L;
  const int prev = (e == 0) ? -1 : (int)keys[e - 1];
  for (int v = prev + 1; v <= seg; ++v) seg_off[v] = e;
  if (e == M - 1)
    for (int v = seg + 1; v <= segments; ++v) seg_off[v] = M;
}

// append every segment longer than `threshold` to `list` (order is irrelevant: each is reduced independently)
__global__ void plan_heavy_kernel(const int32_t* __restrict__ seg_off, int nseg, int threshold, int32_t* __restrict__ list,
                                  int* __restrict__ count) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nseg) return;
  if (seg_off[v + 1] - seg_off[v] > threshold) list[atomicAdd(count, 1)] = v;
}

// ---- compact (source, type) pair table ----
__global__ void pair_mark_kernel(const int32_t* __restrict__ e_src, const int32_t* __restrict__ e_type, int M, int V,
                                 int32_t* __restrict__ used) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < M) used[(size_t)e_type[e] * V + e_src[e]] = 1;   // benign race: every writer stores 1
}
__global__ void pair_fill_kernel(const int32_t* __restrict__ rank, int V, long VL, int32_t* __restrict__ pair_src) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < VL && rank[i + 1] > rank[i]) pair_src[rank[i]] = (int32_t)(i % V);
}
__global__ void pair_edge_kernel(const int32_t* __restrict__ e_src, const int32_t* __restrict__ e_type, int M, int V,
                                 const int32_t* __restrict__ rank, int32_t* __restrict__ e_pair) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < M) e_pair[e] = rank[(size_t)e_type[e] * V + e_src[e]];
}
__global__ void pair_offsets_kernel(const int32_t* __restrict__ rank, int V, int L, int32_t* __restrict__ off) {
  const int l = threadIdx.x;
  if (l <= L) off[l] = rank[(size_t)l * V];
}

// forward plan: heavy targets AND their work items (RGNN_HEAVY_CHUNK edges each) for the multi-CTA split
__global__ void plan_heavy_split_kernel(const int32_t* __restrict__ seg_off, int nseg, int threshold, int chunk,
                                        int32_t* __restrict__ list, int32_t* __restrict__ base_of, int2* __restrict__ items,
                                        int items_cap, int* __restrict__ count, int* __restrict__ item_count) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nseg) return;
  const int deg = seg_off[v + 1] - seg_off[v];
  if (deg <= threshold) return;
  const int n = (deg + chunk - 1) / chunk;
  const int base = atomicAdd(item_count, n);
  const int i = atomicAdd(count, 1);
  list[i] = v;
  base_of[i] = base;
  for (int c = 0; c < n; ++c)
    if (base + c < items_cap) items[base + c] = make_int2(v, c);
}

void ensure_pool_config(int device) {
  static bool done[64] = {false};
  if (device < 0 || device >= 64 || done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t keep = UINT64_MAX;   // never trim: per-batch plan buffers are recycled from the pool
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  done[device] = true;
}

int bits_for(uint64_t n) {   // number of low bits needed to represent values < n
  int b = 1;
  while (b < 32 && (1ull << b) < n) ++b;
  return b;
}

}  // namespace

int plan_ensure_reverse(rgnn_plan* plan, cudaStream_t stream) {
  if (plan->rev_seg_off != nullptr) return RGNN_OK;
  // Inside a capture the allocation below would be a graph allocation, unbacked and unfilled until the graph is replayed,
  // yet kept by the plan for every later (eager) backward: refuse before anything is recorded.
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  RGNN_CHECK_CUDA(cudaStreamIsCapturing(stream, &cap));
  RGNN_REQUIRE(cap == cudaStreamCaptureStatusNone,
               "backward: the first backward on a plan builds its reverse index, which cannot happen during CUDA-graph "
               "capture (run one backward on this plan eagerly before capturing)");
  const int V = plan->V, L = plan->L;
  const int M = (int)plan->M;
  const size_t segments = (size_t)V * L;
  const size_t off_bytes = align_up(sizeof(int32_t) * (segments + 1), 256);
  const size_t m_bytes = align_up(sizeof(int32_t) * (size_t)(M > 0 ? M : 1), 256);
  RGNN_CHECK_CUDA(cudaMallocAsync(&plan->rev_block, off_bytes + 2 * m_bytes + off_bytes, stream));
  char* b = static_cast<char*>(plan->rev_block);
  plan->rev_heavy_list = reinterpret_cast<int32_t*>(b + off_bytes + 2 * m_bytes);
  RGNN_CHECK_CUDA(cudaMemsetAsync(plan->err_flag + 2, 0, sizeof(int), stream));
  plan->rev_src = reinterpret_cast<int32_t*>(b + off_bytes);
  plan->rev_type = reinterpret_cast<int32_t*>(b + off_bytes + m_bytes);
  int32_t* seg_off = reinterpret_cast<int32_t*>(b);
  if (M == 0) {
    RGNN_CHECK_CUDA(cudaMemsetAsync(seg_off, 0, sizeof(int32_t) * (segments + 1), stream));
    plan->rev_seg_off = seg_off;
    return RGNN_OK;
  }
  const int end_bit = bits_for((uint64_t)segments);
  size_t cub_bytes = 0;
  {
    cub::DoubleBuffer<uint32_t> dk(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
    RGNN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, dk, dv, M, 0, end_bit, stream));
  }
  const size_t arr = align_up(sizeof(uint32_t) * (size_t)M, 256);
  char* scratch = nullptr;
  RGNN_CHECK_CUDA(cudaMallocAsync(&scratch, 4 * arr + align_up(cub_bytes, 256), stream));
  uint32_t* k0 = reinterpret_cast<uint32_t*>(scratch);
  uint32_t* k1 = reinterpret_cast<uint32_t*>(scratch + arr);
  int32_t* v0 = reinterpret_cast<int32_t*>(scratch + 2 * arr);
  int32_t* v1 = reinterpret_cast<int32_t*>(scratch + 3 * arr);
  TypeOffsets to;
  for (int l = 0; l <= L; ++l) to.off[l] = plan->type_off[l];
  plan_rev_keys_kernel<<<dim3((plan->max_type_edges + 255) / 256, L), 256, 0, stream>>>(to, L, plan->o_src, k0, v0);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  cub::DoubleBuffer<uint32_t> dk(k0, k1);
  cub::DoubleBuffer<int32_t> dv(v0, v1);
  RGNN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(scratch + 4 * arr, cub_bytes, dk, dv, M, 0, end_bit, stream));
  plan_rev_finalize_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(dk.Current(), dv.Current(), plan->o_tgt,
                                                                           (int)segments, L, M, seg_off, plan->rev_src,
                                                                           plan->rev_type);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  plan_heavy_kernel<<<(unsigned)((segments + 255) / 256), 256, 0, stream>>>(seg_off, (int)segments, RGNN_HEAVY_SEGMENT,
                                                                         plan->rev_heavy_list, plan->err_flag + 2);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  RGNN_CHECK_CUDA(cudaFreeAsync(scratch, stream));
  plan->rev_seg_off = seg_off;
  return RGNN_OK;
}

}  // namespace rgnn

using namespace rgnn;

extern "C" int rgnn_plan_set_num_targets(rgnn_plan_t* plan, int32_t num_targets) {
  RGNN_REQUIRE(plan != nullptr, "plan_set_num_targets: plan is NULL");
  RGNN_REQUIRE(num_targets >= 0 && num_targets <= plan->V, "plan_set_num_targets: %d outside [0, V=%d]", num_targets, plan->V);
  plan->Vt = num_targets;
  return RGNN_OK;
}

extern "C" int rgnn_plan_create(rgnn_plan_t** out, int32_t num_nodes, int32_t num_edge_types,
                                const int32_t* const* adjacency_lists, const int64_t* num_edges, void* stream_) {
  return rgnn_plan_create_ex(out, num_nodes, num_edge_types, adjacency_lists, num_edges, 0, stream_);
}

extern "C" int rgnn_plan_create_ex(rgnn_plan_t** out, int32_t num_nodes, int32_t num_edge_types,
                                   const int32_t* const* adjacency_lists, const int64_t* num_edges, int flags,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool deferred = (flags & RGNN_PLAN_DEFERRED_CHECK) != 0;
  RGNN_REQUIRE(out != nullptr, "plan_create: out is NULL");
  *out = nullptr;
  RGNN_REQUIRE(num_nodes >= 0, "plan_create: num_nodes %d < 0", num_nodes);
  RGNN_REQUIRE(num_edge_types >= 1 && num_edge_types <= RGNN_MAX_EDGE_TYPES,
               "plan_create: num_edge_types %d outside [1, %d]", num_edge_types, RGNN_MAX_EDGE_TYPES);
  RGNN_REQUIRE(adjacency_lists != nullptr && num_edges != nullptr, "plan_create: NULL adjacency table");
  RGNN_REQUIRE((uint64_t)num_nodes * (uint64_t)num_edge_types < (1ull << 32), "plan_create: V*L must be < 2^32");
  if (!deferred) {   // the validated build synchronises the stream, which would invalidate a capture halfway through
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    RGNN_CHECK_CUDA(cudaStreamIsCapturing(stream, &cap));
    RGNN_REQUIRE(cap == cudaStreamCaptureStatusNone,
                 "plan_create: a validated build synchronises the stream and cannot be captured into a CUDA graph "
                 "(build with RGNN_PLAN_DEFERRED_CHECK inside a capture)");
  }

  AdjTable tab;
  int64_t M = 0;
  int32_t maxE = 0;
  rgnn_plan* plan = new (std::nothrow) rgnn_plan();
  RGNN_REQUIRE(plan != nullptr, "plan_create: out of host memory");
  for (int l = 0; l < num_edge_types; ++l) {
    if (num_edges[l] < 0 || (num_edges[l] > 0 && adjacency_lists[l] == nullptr) ||
        (num_edges[l] > 0 && (reinterpret_cast<uintptr_t>(adjacency_lists[l]) & 7u))) {
      delete plan;
      set_error("plan_create: adjacency list %d is NULL / misaligned / negative length", l);
      return RGNN_E_INVALID;
    }
    tab.adj[l] = adjacency_lists[l];
    tab.count[l] = (int32_t)num_edges[l];
    tab.off[l] = (int32_t)M;
    plan->type_off[l] = (int32_t)M;
    M += num_edges[l];
    if (M >= (1ll << 31)) {
      delete plan;
      set_error("plan_create: more than 2^31 messages");
      return RGNN_E_UNSUPPORTED;
    }
    if (num_edges[l] > maxE) maxE = (int32_t)num_edges[l];
  }
  plan->type_off[num_edge_types] = (int32_t)M;
  plan->V = num_nodes;
  plan->Vt = num_nodes; plan->L = num_edge_types; plan->M = M; plan->max_type_edges = maxE;
  cudaGetDevice(&plan->device);

  auto fail = [&](int code) {
    rgnn_plan_destroy(plan);
    return code;
  };
#define PLAN_CUDA(expr)                                                                                    \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return fail(RGNN_E_CUDA);                                                                            \
    }                                                                                                      \
  } while (0)

  // one stream-ordered pool allocation holds every plan array (fast after the first batch: the
  // pool keeps its memory, see ensure_pool_config)
  ensure_pool_config(plan->device);
  const size_t Mz = (size_t)(M > 0 ? M : 1);
  const size_t off_bytes = align_up(sizeof(int32_t) * ((size_t)num_nodes + 1), 256);
  const size_t m_bytes = align_up(sizeof(int32_t) * Mz, 256);
  plan->stream = stream;
  plan->heavy_items_cap = (int32_t)(3 * Mz / (2 * RGNN_HEAVY_CHUNK) + 2);
  const size_t items_bytes = align_up(sizeof(int2) * (size_t)plan->heavy_items_cap, 256);
  PLAN_CUDA(cudaMallocAsync(&plan->block, off_bytes + 5 * m_bytes + 256 + 2 * off_bytes + items_bytes, stream));
  {
    char* b = static_cast<char*>(plan->block);
    plan->seg_off = reinterpret_cast<int32_t*>(b);
    plan->e_src = reinterpret_cast<int32_t*>(b + off_bytes);
    plan->e_type = reinterpret_cast<int32_t*>(b + off_bytes + m_bytes);
    plan->e_orig = reinterpret_cast<int32_t*>(b + off_bytes + 2 * m_bytes);
    plan->o_src = reinterpret_cast<int32_t*>(b + off_bytes + 3 * m_bytes);
    plan->o_tgt = reinterpret_cast<int32_t*>(b + off_bytes + 4 * m_bytes);
    plan->err_flag = reinterpret_cast<int*>(b + off_bytes + 5 * m_bytes);
    plan->heavy_list = reinterpret_cast<int32_t*>(b + off_bytes + 5 * m_bytes + 256);
    plan->heavy_base = reinterpret_cast<int32_t*>(b + off_bytes + 5 * m_bytes + 256 + off_bytes);
    plan->heavy_items = reinterpret_cast<int32_t*>(b + off_bytes + 5 * m_bytes + 256 + 2 * off_bytes);
  }
  PLAN_CUDA(cudaMemsetAsync(plan->err_flag, 0, 4 * sizeof(int), stream));

  if (M == 0) {
    PLAN_CUDA(cudaMemsetAsync(plan->seg_off, 0, sizeof(int32_t) * ((size_t)num_nodes + 1), stream));
    plan->num_heavy_host = 0;
    plan->num_heavy_items_host = 0;
    if (!deferred) PLAN_CUDA(cudaStreamSynchronize(stream));
    *out = plan;
    return RGNN_OK;
  }

  // scratch: keys/vals double buffers + error flag + CUB temp, one allocation
  const int end_bit = bits_for((uint64_t)num_nodes * (uint64_t)num_edge_types);
  size_t cub_bytes = 0;
  {
    cub::DoubleBuffer<uint32_t> dk(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
    PLAN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, dk, dv, (int)M, 0, end_bit, stream));
  }
  const size_t arr = align_up(sizeof(uint32_t) * Mz, 256);
  const size_t total = 4 * arr + align_up(cub_bytes, 256);
  char* scratch = nullptr;
  PLAN_CUDA(cudaMallocAsync(&scratch, total, stream));
  uint32_t* k0 = reinterpret_cast<uint32_t*>(scratch);
  uint32_t* k1 = reinterpret_cast<uint32_t*>(scratch + arr);
  int32_t* v0 = reinterpret_cast<int32_t*>(scratch + 2 * arr);
  int32_t* v1 = reinterpret_cast<int32_t*>(scratch + 3 * arr);
  int* err = plan->err_flag;
  void* cub_tmp = scratch + 4 * arr;

  auto fail_scratch = [&](int code) {
    cudaFreeAsync(scratch, stream);
    cudaStreamSynchronize(stream);
    return fail(code);
  };
#define PLAN_CUDA2(expr)                                                                                   \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return fail_scratch(RGNN_E_CUDA);                                                                    \
    }                                                                                                      \
  } while (0)

  {
    dim3 grid((maxE + 255) / 256, num_edge_types);
    plan_concat_kernel<<<grid, 256, 0, stream>>>(tab, num_nodes, num_edge_types, plan->o_src, plan->o_tgt, k0, v0, err);
    PLAN_CUDA2(cudaGetLastError());
    count_launch();
  }
  cub::DoubleBuffer<uint32_t> dk(k0, k1);
  cub::DoubleBuffer<int32_t> dv(v0, v1);
  PLAN_CUDA2(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, dk, dv, (int)M, 0, end_bit, stream));
  {
    plan_finalize_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(
        dk.Current(), dv.Current(), plan->o_src, num_nodes, num_edge_types, (int)M, plan->seg_off, plan->e_src,
        plan->e_type, plan->e_orig);
    PLAN_CUDA2(cudaGetLastError());
    count_launch();
  }
  if (num_nodes > 0) {
    plan_heavy_split_kernel<<<(num_nodes + 255) / 256, 256, 0, stream>>>(plan->seg_off, num_nodes, RGNN_HEAVY_SEGMENT, RGNN_HEAVY_CHUNK,
                                                                        plan->heavy_list, plan->heavy_base,
                                                                        reinterpret_cast<int2*>(plan->heavy_items), plan->heavy_items_cap,
                                                                        plan->err_flag + 1, plan->err_flag + 3);
    PLAN_CUDA2(cudaGetLastError());
    count_launch();
  }
  // compact (source, type) pair table for sparsely typed graphs (see plan.cuh)
  const size_t VL = (size_t)num_nodes * num_edge_types;
  if ((double)M < 0.75 * (double)VL) {
    const size_t rank_bytes = align_up(sizeof(int32_t) * (VL + 1), 256);
    size_t scan_bytes = 0;
    PLAN_CUDA2(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(VL + 1), stream));
    scan_bytes = align_up(scan_bytes, 256);
    PLAN_CUDA2(cudaMallocAsync(&plan->pair_block, 2 * m_bytes + align_up(sizeof(int32_t) * (RGNN_MAX_EDGE_TYPES + 1), 256), stream));
    char* pb = static_cast<char*>(plan->pair_block);
    plan->pair_src = reinterpret_cast<int32_t*>(pb);
    plan->e_pair = reinterpret_cast<int32_t*>(pb + m_bytes);
    plan->pair_off_dev = reinterpret_cast<int32_t*>(pb + 2 * m_bytes);
    char* tmp = nullptr;
    PLAN_CUDA2(cudaMallocAsync(&tmp, rank_bytes + scan_bytes, stream));
    int32_t* rank = reinterpret_cast<int32_t*>(tmp);
    cudaError_t pe = cudaMemsetAsync(rank, 0, sizeof(int32_t) * (VL + 1), stream);
    if (pe == cudaSuccess) {
      pair_mark_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(plan->e_src, plan->e_type, (int)M, num_nodes, rank);
      pe = cub::DeviceScan::ExclusiveSum(tmp + rank_bytes, scan_bytes, rank, rank, (int)(VL + 1), stream);
    }
    if (pe == cudaSuccess) {
      pair_fill_kernel<<<(unsigned)((VL + 255) / 256), 256, 0, stream>>>(rank, num_nodes, (long)VL, plan->pair_src);
      pair_edge_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(plan->e_src, plan->e_type, (int)M, num_nodes, rank, plan->e_pair);
      pair_offsets_kernel<<<1, RGNN_MAX_EDGE_TYPES + 1, 0, stream>>>(rank, num_nodes, num_edge_types, plan->pair_off_dev);
      pe = cudaGetLastError();
      count_launch(5);
    }
    cudaFreeAsync(tmp, stream);
    PLAN_CUDA2(pe);
  }
  PLAN_CUDA2(cudaFreeAsync(scratch, stream));
  if (!deferred) {
    const int rc = rgnn_plan_status(plan);
    if (rc != RGNN_OK) return fail(rc);
  }
  *out = plan;
  return RGNN_OK;
#undef PLAN_CUDA
#undef PLAN_CUDA2
}

extern "C" int rgnn_plan_status(const rgnn_plan_t* plan) {
  RGNN_REQUIRE(plan != nullptr, "plan_status: plan is NULL");
  if (plan->err_flag == nullptr) return RGNN_OK;
  {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    RGNN_CHECK_CUDA(cudaStreamIsCapturing(plan->stream, &cap));
    RGNN_REQUIRE(cap == cudaStreamCaptureStatusNone,
                 "plan_status: synchronises the plan's creation stream, which is capturing a CUDA graph (call it after "
                 "the capture, once the graph has been replayed)");
  }
  int flags[4] = {0, 0, 0, 0};
  RGNN_CHECK_CUDA(cudaMemcpyAsync(flags, plan->err_flag, 4 * sizeof(int), cudaMemcpyDeviceToHost, plan->stream));
  rgnn_plan* mp = const_cast<rgnn_plan*>(plan);
  if (plan->pair_off_dev != nullptr && plan->n_pairs < 0)
    RGNN_CHECK_CUDA(cudaMemcpyAsync(mp->pair_type_off, plan->pair_off_dev, sizeof(int32_t) * (plan->L + 1), cudaMemcpyDeviceToHost, plan->stream));
  RGNN_CHECK_CUDA(cudaStreamSynchronize(plan->stream));
  if (plan->pair_off_dev != nullptr && plan->n_pairs < 0) {
    mp->n_pairs = mp->pair_type_off[plan->L];
    mp->max_type_pairs = 0;
    for (int l = 0; l < plan->L; ++l)
      if (mp->pair_type_off[l + 1] - mp->pair_type_off[l] > mp->max_type_pairs) mp->max_type_pairs = mp->pair_type_off[l + 1] - mp->pair_type_off[l];
  }
  const_cast<rgnn_plan*>(plan)->num_heavy_host = flags[1];
  const_cast<rgnn_plan*>(plan)->num_heavy_items_host = flags[3];
  const int herr = flags[0];
  if (herr != 0) {
    set_error("plan: adjacency list holds a node index outside [0, %d)", plan->V);
    return RGNN_E_INVALID;
  }
  return RGNN_OK;
}

extern "C" int rgnn_plan_destroy(rgnn_plan_t* plan) {
  if (plan == nullptr) return RGNN_OK;
  if (plan->rev_block != nullptr) cudaFreeAsync(plan->rev_block, plan->stream);
  if (plan->pair_block != nullptr) cudaFreeAsync(plan->pair_block, plan->stream);
  // stream-ordered on the creation stream: safe after work queued on THAT stream; work on other streams must be ordered
  // before this call by the caller (include/rgnn.h "threads")
  if (plan->block != nullptr) cudaFreeAsync(plan->block, plan->stream);
  delete plan;
  return RGNN_OK;
}

extern "C" int32_t rgnn_plan_num_nodes(const rgnn_plan_t* plan) { return plan ? plan->V : -1; }
extern "C" int32_t rgnn_plan_num_edge_types(const rgnn_plan_t* plan) { return plan ? plan->L : -1; }
extern "C" int64_t rgnn_plan_num_edges(const rgnn_plan_t* plan) { return plan ? plan->M : -1; }

extern "C" int rgnn_plan_export(const rgnn_plan_t* plan, int32_t* seg_off, int32_t* e_src, int32_t* e_type,
                                int32_t* e_orig, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(plan != nullptr, "plan_export: plan is NULL");
  const size_t mb = sizeof(int32_t) * (size_t)plan->M;
  if (seg_off) RGNN_CHECK_CUDA(cudaMemcpyAsync(seg_off, plan->seg_off, sizeof(int32_t) * ((size_t)plan->V + 1), cudaMemcpyDeviceToDevice, stream));
  if (e_src && mb) RGNN_CHECK_CUDA(cudaMemcpyAsync(e_src, plan->e_src, mb, cudaMemcpyDeviceToDevice, stream));
  if (e_type && mb) RGNN_CHECK_CUDA(cudaMemcpyAsync(e_type, plan->e_type, mb, cudaMemcpyDeviceToDevice, stream));
  if (e_orig && mb) RGNN_CHECK_CUDA(cudaMemcpyAsync(e_orig, plan->e_orig, mb, cudaMemcpyDeviceToDevice, stream));
  return RGNN_OK;
}
