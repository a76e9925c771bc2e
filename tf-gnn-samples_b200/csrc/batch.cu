// batch.cu -- pack one minibatch on the device from a device-resident graph set.
//
// The task batchers (tasks/ppi_task.py:213-251, tasks/qm9_task.py:216-256) loop over the graphs of a batch on the host, shift
// every edge list by the graph's node offset and concatenate features, edge lists and in-degrees.  Here the whole data set
// lives on the device once, concatenated in data-set order with graph-local node ids (CSR over graphs), and a batch -- the
// graphs order[start, start + n) -- is gathered by three kernels:
//   pack_offsets_kernel  one CTA per count array (nodes, then every edge type): gathers the per-graph counts in batch order
//                        and exclusive-scans them (cub::BlockScan, running prefix) into the batch's offsets; CTA 0 also
//                        gathers the per-graph tensors.  Each CTA compares its total with the caller's.
//   pack_nodes_kernel    one CTA per tile of output rows: a binary search over the batch's node offsets finds each row's
//                        graph, then the CTA copies every per-node tensor, the in-degrees and the graph ids of the tile.
//   pack_edges_kernel    one thread per output edge of every type, found by binary search over that type's batch offsets:
//                        the source edge shifted by its graph's batch node offset.
// Every output element has one writer (no atomics), edges keep batch-graph order then the graph's own order (what
// pack_batch produces), values are copied, so the result is bit-identical to the host packer.  Output indices are bounded
// by the caller's totals, never by the device-computed ones, so a wrong total cannot write past a buffer.
#include "common.cuh"

#include <cub/block/block_scan.cuh>

namespace rgnn {

namespace {

constexpr int PACK_SCAN_THREADS = 512;
constexpr int PACK_SCAN_ITEMS = 4;                     // per thread and pass: 2048 graphs per pass of the scan
constexpr int PACK_TILE_ROWS = 64;
constexpr int PACK_NODE_THREADS = 256;
constexpr int PACK_EDGE_THREADS = 256;

struct PackSet {
  const int64_t* node_off;                              // [G + 1]
  const int64_t* edge_off[RGNN_MAX_EDGE_TYPES];         // [G + 1] per type
  const int32_t* edges[RGNN_MAX_EDGE_TYPES];            // [E_l, 2] per type, graph-local ids
  const float* indeg;                                   // [L, N]
  const float* node_t[RGNN_PACK_MAX_TENSORS];           // [N, w_k]
  int32_t node_w[RGNN_PACK_MAX_TENSORS];
  const float* graph_t[RGNN_PACK_MAX_TENSORS];          // [T_k, G]
  int32_t graph_rows[RGNN_PACK_MAX_TENSORS];
  int64_t G, N;
  int32_t L, num_node_t, num_graph_t;
};

struct PackOut {
  int32_t* adj[RGNN_MAX_EDGE_TYPES];                    // [E_l, 2]
  int64_t E[RGNN_MAX_EDGE_TYPES];                       // caller's totals
  float* node_t[RGNN_PACK_MAX_TENSORS];                 // [V, w_k]
  float* graph_t[RGNN_PACK_MAX_TENSORS];                // [T_k, n]
  float* indeg;                                         // [L, V]
  int32_t* graph_nodes_list;                            // [V] or NULL
  int32_t V;
};

// workspace: offsets int64 [(1 + L) x (n + 1)] (array 0 = nodes, 1 + l = edges of type l), then int32 flags [1 + L + 1]
// (mismatch of array k, then "order entry outside [0, G)")
size_t offsets_bytes(int64_t n, int L) { return align_up(sizeof(int64_t) * (size_t)(1 + L) * (size_t)(n + 1), 256); }
size_t flags_bytes(int L) { return align_up(sizeof(int32_t) * (size_t)(L + 2), 256); }

// grid = 1 + L CTAs.  offs[k * (n + 1) + i] = sum of the counts of batch graphs [0, i) in array k.
__global__ void __launch_bounds__(PACK_SCAN_THREADS)
pack_offsets_kernel(const __grid_constant__ PackSet s, const __grid_constant__ PackOut o, const int32_t* __restrict__ order,
                    int64_t start, int n, int64_t* __restrict__ offs, int32_t* __restrict__ flags) {
  using Scan = cub::BlockScan<int64_t, PACK_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int64_t carry;
  const int k = blockIdx.x;
  const int64_t* off = k == 0 ? s.node_off : s.edge_off[k - 1];
  int64_t* out = offs + (size_t)k * (n + 1);
  int bad_order = 0;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += PACK_SCAN_THREADS * PACK_SCAN_ITEMS) {
    int64_t c[PACK_SCAN_ITEMS], excl[PACK_SCAN_ITEMS], total;
#pragma unroll
    for (int j = 0; j < PACK_SCAN_ITEMS; ++j) {          // blocked: thread t holds items [t * ITEMS, (t + 1) * ITEMS)
      const int i = base + threadIdx.x * PACK_SCAN_ITEMS + j;
      c[j] = 0;
      if (i < n) {
        const int64_t g = order[start + i];
        if (g >= 0 && g < s.G) {
          c[j] = off[g + 1] - off[g];
          if (k == 0)
            for (int t = 0; t < s.num_graph_t; ++t)
              for (int r = 0; r < s.graph_rows[t]; ++r) o.graph_t[t][(size_t)r * n + i] = s.graph_t[t][r * s.G + g];
        } else {
          bad_order = 1;
        }
      }
    }
    Scan(tmp).ExclusiveSum(c, excl, total);
#pragma unroll
    for (int j = 0; j < PACK_SCAN_ITEMS; ++j) {
      const int i = base + threadIdx.x * PACK_SCAN_ITEMS + j;
      if (i < n) out[i] = carry + excl[j];
    }
    __syncthreads();                                     // every thread has read carry and tmp
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  const int any_bad = __syncthreads_or(bad_order);
  if (threadIdx.x == 0) {
    out[n] = carry;
    const int64_t want = k == 0 ? (int64_t)o.V : o.E[k - 1];
    flags[k] = carry != want;
    if (k == 0) flags[1 + s.L] = any_bad;
  }
}

// largest i in [0, n) with off[i] <= x (off ascending, off[0] = 0 <= x)
__device__ __forceinline__ int find_graph(const int64_t* __restrict__ off, int n, int64_t x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// grid = max(1, ceil(V / PACK_TILE_ROWS)).  CTA 0 also folds the offset kernel's flags into the caller's status word.
__global__ void __launch_bounds__(PACK_NODE_THREADS)
pack_nodes_kernel(const __grid_constant__ PackSet s, const __grid_constant__ PackOut o, const int32_t* __restrict__ order,
                  int64_t start, int n, const int64_t* __restrict__ offs, const int32_t* __restrict__ flags,
                  int32_t* __restrict__ status) {
  __shared__ int64_t src_row[PACK_TILE_ROWS];              // -1: row not written
  if (blockIdx.x == 0 && threadIdx.x == 0 && status != nullptr) {
    int st = flags[0] ? RGNN_PACK_NODES_MISMATCH : 0;
    for (int l = 0; l < s.L; ++l) st |= flags[1 + l] ? RGNN_PACK_EDGES_MISMATCH : 0;
    st |= flags[1 + s.L] ? RGNN_PACK_BAD_ORDER : 0;
    *status = st;
  }
  const int64_t r0 = (int64_t)blockIdx.x * PACK_TILE_ROWS;
  const int64_t V = o.V;
  if (r0 >= V || n == 0) return;
  const int rows = (int)min((int64_t)PACK_TILE_ROWS, V - r0);
  const int64_t dev_total = offs[n];
  if (threadIdx.x < rows) {
    const int64_t r = r0 + threadIdx.x;
    int64_t src = -1;
    int i = -1;
    if (r < dev_total) {                                 // rows past the device total (wrong caller total) stay unwritten
      i = find_graph(offs, n, r);
      src = s.node_off[order[start + i]] + (r - offs[i]);
    }
    src_row[threadIdx.x] = src;
    if (o.graph_nodes_list != nullptr && i >= 0) o.graph_nodes_list[r] = i;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < s.L * rows; idx += PACK_NODE_THREADS) {
    const int l = idx / rows, t = idx - l * rows;
    const int64_t src = src_row[t];
    if (src >= 0) o.indeg[(size_t)l * V + r0 + t] = s.indeg[(size_t)l * s.N + src];
  }
  for (int k = 0; k < s.num_node_t; ++k) {
    const int w = s.node_w[k];
    const float* __restrict__ in = s.node_t[k];
    float* __restrict__ out = o.node_t[k] + (size_t)r0 * w;
    for (int idx = threadIdx.x; idx < rows * w; idx += PACK_NODE_THREADS) {
      const int t = idx / w, c = idx - t * w;
      const int64_t src = src_row[t];
      if (src >= 0) out[idx] = in[(size_t)src * w + c];
    }
  }
}

// grid = (ceil(max_l E_l / PACK_EDGE_THREADS), L), E_l the caller's totals
__global__ void __launch_bounds__(PACK_EDGE_THREADS)
pack_edges_kernel(const __grid_constant__ PackSet s, const __grid_constant__ PackOut o, const int32_t* __restrict__ order,
                  int64_t start, int n, const int64_t* __restrict__ offs) {
  const int l = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * PACK_EDGE_THREADS + threadIdx.x;
  if (e >= o.E[l] || n == 0) return;
  const int64_t* __restrict__ eoff = offs + (size_t)(1 + l) * (n + 1);
  if (e >= eoff[n]) return;                              // past the device total: the caller's total was too large
  const int i = find_graph(eoff, n, e);
  const int64_t g = order[start + i];
  const int2 v = __ldg(reinterpret_cast<const int2*>(s.edges[l]) + (s.edge_off[l][g] + (e - eoff[i])));
  const int32_t shift = (int32_t)__ldg(offs + i);       // the graph's first node in the batch
  reinterpret_cast<int2*>(o.adj[l])[e] = make_int2(v.x + shift, v.y + shift);
}

}  // namespace

}  // namespace rgnn

using namespace rgnn;

extern "C" size_t rgnn_pack_workspace_bytes(int32_t num_batch_graphs, int32_t num_edge_types) {
  if (num_batch_graphs < 0 || num_edge_types < 1 || num_edge_types > RGNN_MAX_EDGE_TYPES) return 0;
  return offsets_bytes(num_batch_graphs, num_edge_types) + flags_bytes(num_edge_types);
}

extern "C" int rgnn_pack_minibatch(int64_t num_graphs, int64_t num_nodes, int32_t num_edge_types,
                                   const int64_t* node_offsets, const int64_t* const* edge_offsets,
                                   const int32_t* const* adjacency_lists, const float* num_incoming,
                                   int32_t num_node_tensors, const float* const* node_tensors, const int32_t* node_widths,
                                   int32_t num_graph_tensors, const float* const* graph_tensors, const int32_t* graph_rows,
                                   const int32_t* order, int64_t start, int32_t num_batch_graphs, int32_t batch_nodes,
                                   const int64_t* batch_edges, float* const* out_node_tensors,
                                   int32_t* const* out_adjacency_lists, float* out_num_incoming,
                                   int32_t* out_graph_nodes_list, float* const* out_graph_tensors, int32_t* status,
                                   void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int L = num_edge_types, n = num_batch_graphs;
  RGNN_REQUIRE(num_graphs >= 0 && num_nodes >= 0, "pack_minibatch: negative graph-set size (G=%lld, N=%lld)",
               (long long)num_graphs, (long long)num_nodes);
  RGNN_REQUIRE(L >= 1 && L <= RGNN_MAX_EDGE_TYPES, "pack_minibatch: num_edge_types %d outside [1, %d]", L,
               RGNN_MAX_EDGE_TYPES);
  RGNN_REQUIRE(start >= 0 && n >= 0 && batch_nodes >= 0, "pack_minibatch: negative start / batch size / node total");
  RGNN_REQUIRE(num_node_tensors >= 0 && num_node_tensors <= RGNN_PACK_MAX_TENSORS && num_graph_tensors >= 0 &&
               num_graph_tensors <= RGNN_PACK_MAX_TENSORS,
               "pack_minibatch: %d per-node / %d per-graph tensors (at most %d each)", num_node_tensors, num_graph_tensors,
               RGNN_PACK_MAX_TENSORS);
  RGNN_REQUIRE(node_offsets != nullptr && edge_offsets != nullptr && adjacency_lists != nullptr && batch_edges != nullptr &&
               out_adjacency_lists != nullptr, "pack_minibatch: NULL graph-set or adjacency table");
  RGNN_REQUIRE(n == 0 || order != nullptr, "pack_minibatch: order is NULL");
  RGNN_REQUIRE(batch_nodes == 0 || (num_incoming != nullptr && out_num_incoming != nullptr),
               "pack_minibatch: NULL in-degree buffer");
  PackSet s = {};
  PackOut o = {};
  s.node_off = node_offsets; s.indeg = num_incoming; s.G = num_graphs; s.N = num_nodes; s.L = L;
  s.num_node_t = num_node_tensors; s.num_graph_t = num_graph_tensors;
  o.indeg = out_num_incoming; o.graph_nodes_list = out_graph_nodes_list; o.V = batch_nodes;
  int64_t maxE = 0;
  for (int l = 0; l < L; ++l) {
    RGNN_REQUIRE(batch_edges[l] >= 0 && batch_edges[l] < (1ll << 31), "pack_minibatch: edge total of type %d is %lld", l,
                 (long long)batch_edges[l]);
    RGNN_REQUIRE(edge_offsets[l] != nullptr, "pack_minibatch: edge offsets of type %d are NULL", l);
    RGNN_REQUIRE(batch_edges[l] == 0 || (adjacency_lists[l] != nullptr && out_adjacency_lists[l] != nullptr &&
                                         (reinterpret_cast<uintptr_t>(adjacency_lists[l]) & 7u) == 0 &&
                                         (reinterpret_cast<uintptr_t>(out_adjacency_lists[l]) & 7u) == 0),
                 "pack_minibatch: adjacency list of type %d is NULL or not 8-byte aligned", l);
    s.edge_off[l] = edge_offsets[l]; s.edges[l] = adjacency_lists[l];
    o.adj[l] = out_adjacency_lists[l]; o.E[l] = batch_edges[l];
    if (batch_edges[l] > maxE) maxE = batch_edges[l];
  }
  if (num_node_tensors > 0)
    RGNN_REQUIRE(node_tensors != nullptr && node_widths != nullptr && out_node_tensors != nullptr,
                 "pack_minibatch: NULL per-node tensor table");
  for (int k = 0; k < num_node_tensors; ++k) {
    RGNN_REQUIRE(node_widths[k] >= 1, "pack_minibatch: per-node tensor %d has width %d", k, node_widths[k]);
    RGNN_REQUIRE(batch_nodes == 0 || (node_tensors[k] != nullptr && out_node_tensors[k] != nullptr),
                 "pack_minibatch: per-node tensor %d is NULL", k);
    s.node_t[k] = node_tensors[k]; s.node_w[k] = node_widths[k]; o.node_t[k] = out_node_tensors[k];
  }
  if (num_graph_tensors > 0)
    RGNN_REQUIRE(graph_tensors != nullptr && graph_rows != nullptr && out_graph_tensors != nullptr,
                 "pack_minibatch: NULL per-graph tensor table");
  for (int k = 0; k < num_graph_tensors; ++k) {
    RGNN_REQUIRE(graph_rows[k] >= 0, "pack_minibatch: per-graph tensor %d has %d rows", k, graph_rows[k]);
    RGNN_REQUIRE(n == 0 || graph_rows[k] == 0 || (graph_tensors[k] != nullptr && out_graph_tensors[k] != nullptr),
                 "pack_minibatch: per-graph tensor %d is NULL", k);
    s.graph_t[k] = graph_tensors[k]; s.graph_rows[k] = graph_rows[k]; o.graph_t[k] = out_graph_tensors[k];
  }
  const size_t need = rgnn_pack_workspace_bytes(n, L);
  RGNN_REQUIRE(aligned16(workspace), "pack_minibatch: workspace is not 16-byte aligned");
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("pack_minibatch: workspace of %zu bytes, %zu needed", workspace ? workspace_bytes : (size_t)0, need);
    return RGNN_E_WORKSPACE;
  }
  int64_t* offs = static_cast<int64_t*>(workspace);
  int32_t* flags = reinterpret_cast<int32_t*>(static_cast<char*>(workspace) + offsets_bytes(n, L));

  pack_offsets_kernel<<<1 + L, PACK_SCAN_THREADS, 0, stream>>>(s, o, order, start, n, offs, flags);
  RGNN_CHECK_CUDA(cudaGetLastError());
  const unsigned tiles = (unsigned)((batch_nodes + PACK_TILE_ROWS - 1) / PACK_TILE_ROWS);
  pack_nodes_kernel<<<tiles > 0 ? tiles : 1, PACK_NODE_THREADS, 0, stream>>>(s, o, order, start, n, offs, flags, status);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  if (maxE > 0 && n > 0) {
    pack_edges_kernel<<<dim3((unsigned)((maxE + PACK_EDGE_THREADS - 1) / PACK_EDGE_THREADS), L), PACK_EDGE_THREADS, 0,
                        stream>>>(s, o, order, start, n, offs);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return RGNN_OK;
}
