// seg_kernels.cu -- the edge stage of every layer as fused sorted-segment kernels.
//
// One warp owns one target node.  Its incoming edges are contiguous in the plan (CSR by target,
// all edge types), so the warp streams the gathered message rows T[src, type, :] with 128-bit
// coalesced loads (one row = D*4 bytes, each lane reads NV float4), applies the per-message
// scale 1/(c+1e-7) / FiLM modulation / activation in registers, reduces in registers, applies
// the layer's epilogue (aggregation divisor, activation, layer norm) and writes the output row
// once.  No [M, D] message matrix, no concat, no atomics, deterministic order.
//
// Replaces: tf.nn.embedding_lookup + scale + tf.concat + tf.unsorted_segment_* + activation
// (gnns/rgcn.py:84-114, ggnn.py:76-90, gnn_film.py:88-120, gnn_edge_mlp.py:87-119,
// rgin.py:106-139), dpu_utils unsorted_segment_log_softmax + per-head weighted segment sums
// (rgat.py:120-138), tf.contrib.layers.layer_norm (A.5).
#include "seg.cuh"

namespace rgnn {

namespace {

constexpr int WARPS_PER_BLOCK = 8;
constexpr int UNROLL = 4;     // message rows in flight per warp

__device__ __forceinline__ float4 f4(float v) { return make_float4(v, v, v, v); }
__device__ __forceinline__ float4 mul4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 max4(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {   // a*b + c
  return make_float4(a.x * b.x + c.x, a.y * b.y + c.y, a.z * b.z + c.z, a.w * b.w + c.w);
}

// tf.contrib.layers.layer_norm over one row held by a warp (A.5): biased variance, eps 1e-12,
// evaluated as x*inv + (beta - mean*inv) with inv = rsqrt(var + eps) * gamma.
template <int NV>
__device__ __forceinline__ void warp_layer_norm(float4 (&x)[NV], const bool (&ok)[NV], int D, int lane,
                                                const float* __restrict__ gamma, const float* __restrict__ beta) {
  float s = 0.0f;
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) s += (x[k].x + x[k].y) + (x[k].z + x[k].w);
  const float mean = warp_sum(s) / (float)D;
  float q = 0.0f;
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) {
      const float a = x[k].x - mean, b = x[k].y - mean, c = x[k].z - mean, d = x[k].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  const float var = warp_sum(q) / (float)D;
  const float rstd = 1.0f / sqrtf(var + 1e-12f);
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) {
      const int col = k * 128 + lane * 4;
      const float4 g = ldg4(gamma + col), b = ldg4(beta + col);
      float inv;
      inv = rstd * g.x; x[k].x = x[k].x * inv + (b.x - mean * inv);
      inv = rstd * g.y; x[k].y = x[k].y * inv + (b.y - mean * inv);
      inv = rstd * g.z; x[k].z = x[k].z * inv + (b.z - mean * inv);
      inv = rstd * g.w; x[k].w = x[k].w * inv + (b.w - mean * inv);
    }
}

// NV float4 per lane (the warp covers 128*NV columns starting at blockIdx.y * 128*NV); MODE = MsgMode;
// MAXAGG = tf.unsorted_segment_max; SCALED = per-message 1/(c+1e-7); ACTMSG = activation applied per message.
// Layer-norm epilogues need the whole row in one warp (gridDim.y == 1).
// Code size matters here: the SM's instruction cache is small, so rare paths are template flags (separate small
// kernels), not runtime branches, and nothing is duplicated.
template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
__device__ __forceinline__ void seg_accumulate(const SegParams& p, int v, int col0, int lane, const bool (&ok)[NV],
                                               int beg, int end, int chunk0, int chunk_stride, float4 (&acc)[NV]) {
  const int act_msg = ACTMSG ? p.act_msg : RGNN_ACT_LINEAR;
  int cur_type = -1;
  float4 m0[NV], m1[NV];   // gamma/beta (FILM) or q (ADDTGT) of the current (v, type) run
#pragma unroll
  for (int k = 0; k < NV; ++k) { m0[k] = f4(1.0f); m1[k] = f4(0.0f); }
  const float* tbase = p.table + col0;

  for (int e0 = beg + 32 * chunk0; e0 < end; e0 += 32 * chunk_stride) {
    const int n = min(32, end - e0);
    int my_type = 0;
    float my_scale = 1.0f;
    long my_off = 0;
    if (lane < n) {
      my_type = __ldg(p.e_type + e0 + lane);
      const int idx = __ldg(p.e_idx + e0 + lane);
      my_off = (long)idx * p.stride_idx + (long)my_type * p.stride_type;
      if (SCALED)   // 1.0f / (c + SMALL_NUMBER) evaluated in fp32 like the reference (rgcn.py:104)
        my_scale = 1.0f / (__ldg(p.num_incoming + (size_t)my_type * p.scale_ld + (p.scale_by_idx ? idx : v)) + 1e-7f);
    }
    for (int j = 0; j < n; j += UNROLL) {
      float4 r[UNROLL][NV];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (j + u < n) {
          const long off = __shfl_sync(0xffffffffu, my_off, j + u);
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (ok[k]) r[u][k] = ldg4(tbase + off + k * 128);
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (j + u < n) {
          const float sc = SCALED ? __shfl_sync(0xffffffffu, my_scale, j + u) : 1.0f;
          if (MODE != MSG_LINEAR) {
            const int ty = __shfl_sync(0xffffffffu, my_type, j + u);
            if (ty != cur_type) {   // warp-uniform: new (v, type) run
              cur_type = ty;
              const float* mrow = p.mod_table + (size_t)v * p.mod_stride_node + (size_t)ty * p.mod_stride_type + col0;
#pragma unroll
              for (int k = 0; k < NV; ++k)
                if (ok[k]) {
                  m0[k] = ldg4(mrow + k * 128);
                  if (MODE == MSG_FILM) m1[k] = ldg4(mrow + p.D + k * 128);
                }
            }
          }
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (ok[k]) {
              float4 m = r[u][k];
              if (MODE == MSG_LINEAR && !MAXAGG && !ACTMSG) {   // hot path: acc += s * t, one FMA / add per element
                if (SCALED) {
                  acc[k].x = fmaf(m.x, sc, acc[k].x); acc[k].y = fmaf(m.y, sc, acc[k].y);
                  acc[k].z = fmaf(m.z, sc, acc[k].z); acc[k].w = fmaf(m.w, sc, acc[k].w);
                } else {
                  acc[k] = add4(acc[k], m);
                }
                continue;
              }
              if (MODE == MSG_LINEAR) {
                if (SCALED) m = mul4(m, sc);
              } else if (MODE == MSG_FILM) {
                if (SCALED) m = mul4(m, sc);
                m = fma4(m0[k], m, m1[k]);
              } else {
                m = add4(m, m0[k]);
                if (SCALED) m = mul4(m, sc);
              }
              if (ACTMSG) m = act4(m, act_msg);
              acc[k] = MAXAGG ? max4(acc[k], m) : add4(acc[k], m);
            }
        }
      }
    }
  }
}

// aggregation divisor (A.2), output activation, optional layer norm, store
template <int NV>
__device__ __forceinline__ void seg_finish(const SegParams& p, int v, int col0, int lane, const bool (&ok)[NV], int count,
                                           float4 (&acc)[NV]) {
  if (p.agg == RGNN_AGG_MEAN || p.agg == RGNN_AGG_SQRT_N) {   // mean = sum / max(n,1); sqrt_n = sum / sqrt(max(n,1))
    const float cnt = fmaxf((float)count, 1.0f);
    const float div = (p.agg == RGNN_AGG_MEAN) ? cnt : sqrtf(cnt);
#pragma unroll
    for (int k = 0; k < NV; ++k)
      acc[k] = make_float4(acc[k].x / div, acc[k].y / div, acc[k].z / div, acc[k].w / div);
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) acc[k] = act4_cold(acc[k], p.act_out);
  if (p.ln_gamma != nullptr) warp_layer_norm<NV>(acc, ok, p.D, lane, p.ln_gamma, p.ln_beta);
  float* orow = p.out + (size_t)v * p.ld_out + col0;
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) *reinterpret_cast<float4*>(orow + k * 128) = acc[k];
}

template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_reduce_kernel(const __grid_constant__ SegParams p) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int col0 = blockIdx.y * (128 * NV) + lane * 4;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);   // plan arrays: not produced by the predecessor kernel
  pdl_wait();                                                             // the table (T) is: wait for the transform GEMM
  pdl_launch_dependents();
  if (p.heavy_threshold > 0 && end - beg > p.heavy_threshold) return;   // left to seg_reduce_heavy_kernel
  bool ok[NV];
  float4 acc[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = (col0 + k * 128) < p.D;
    acc[k] = f4(MAXAGG ? -FLT_MAX : 0.0f);   // empty max segment -> lowest() (A.2)
  }
  seg_accumulate<NV, MODE, MAXAGG, SCALED, ACTMSG>(p, v, col0, lane, ok, beg, end, 0, 1, acc);
  seg_finish<NV>(p, v, col0, lane, ok, end - beg, acc);
}

// Small batches (V * D/128 warps do not fill the SMs: the PPI-shaped single graph has 4,490) can leave the warp-per-128-column
// kernel latency-bound.  Here a warp owns a 64-column
// slice and its two half-warps gather two DIFFERENT edges of the target per load instruction (each 16 lanes x 16 B = 256 B),
// so the same bytes per instruction are in flight from twice as many warps; the two partial sums are combined with one
// xor-16 shuffle round at the end (fixed order: deterministic).  Linear messages, sum / mean / sqrt_n only.
template <bool SCALED>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_reduce_half_kernel(const __grid_constant__ SegParams p) {
  const int lane = threadIdx.x & 31, half = lane >> 4, l16 = lane & 15;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int col0 = blockIdx.y * 64 + l16 * 4;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  pdl_wait();
  pdl_launch_dependents();
  if (p.heavy_threshold > 0 && end - beg > p.heavy_threshold) return;   // left to seg_reduce_heavy_kernel
  const bool okc = col0 < p.D;
  float4 acc = f4(0.0f);
  const float* tbase = p.table + col0;
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    float my_scale = 1.0f;
    long my_off = 0;
    if (lane < n) {
      const int ty = __ldg(p.e_type + e0 + lane);
      const int idx = __ldg(p.e_idx + e0 + lane);
      my_off = (long)idx * p.stride_idx + (long)ty * p.stride_type;
      if (SCALED) my_scale = 1.0f / (__ldg(p.num_incoming + (size_t)ty * p.scale_ld + (p.scale_by_idx ? idx : v)) + 1e-7f);
    }
    for (int j = 0; j < n; j += 2 * UNROLL) {
      float4 r[UNROLL];
      bool valid[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int e = j + 2 * u + half;                 // <= 31
        const long off = __shfl_sync(0xffffffffu, my_off, e);
        valid[u] = okc && e < n;
        if (valid[u]) r[u] = ldg4(tbase + off);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const float sc = SCALED ? __shfl_sync(0xffffffffu, my_scale, j + 2 * u + half) : 1.0f;
        if (valid[u]) {
          if (SCALED) {
            acc.x = fmaf(r[u].x, sc, acc.x); acc.y = fmaf(r[u].y, sc, acc.y);
            acc.z = fmaf(r[u].z, sc, acc.z); acc.w = fmaf(r[u].w, sc, acc.w);
          } else {
            acc = add4(acc, r[u]);
          }
        }
      }
    }
  }
  acc.x += __shfl_xor_sync(0xffffffffu, acc.x, 16); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, 16);
  acc.z += __shfl_xor_sync(0xffffffffu, acc.z, 16); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, 16);
  bool ok1[1] = {okc && half == 0};
  float4 a1[1] = {acc};
  seg_finish<1>(p, v, col0, lane, ok1, end - beg, a1);
}

// Degree skew: a target with thousands of incoming edges would serialise on one warp (Zipf-skewed PPI-shaped
// batch: 1.0 ms instead of 35 us per layer).  Here a whole CTA takes one heavy target: warp w reduces the
// 32-edge chunks w, w+8, ..., the 8 partial rows are combined in a fixed order (still deterministic).
template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_reduce_heavy_kernel(const __grid_constant__ SegParams p) {
  __shared__ float4 part[WARPS_PER_BLOCK][NV][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col0 = blockIdx.y * (128 * NV) + lane * 4;
  const int nheavy = *p.heavy_count;
  bool ok[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) ok[k] = (col0 + k * 128) < p.D;
  for (int i = blockIdx.x; i < nheavy; i += gridDim.x) {
    const int v = __ldg(p.heavy_list + i);
    if (v >= p.V) continue;                             // not a wanted target (rgnn_plan_set_num_targets): row left untouched
    const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
    float4 acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = f4(MAXAGG ? -FLT_MAX : 0.0f);
    seg_accumulate<NV, MODE, MAXAGG, SCALED, ACTMSG>(p, v, col0, lane, ok, beg, end, warp, WARPS_PER_BLOCK, acc);
#pragma unroll
    for (int k = 0; k < NV; ++k) part[warp][k][lane] = acc[k];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        float4 t = part[0][k][lane];
#pragma unroll
        for (int w = 1; w < WARPS_PER_BLOCK; ++w) t = MAXAGG ? max4(t, part[w][k][lane]) : add4(t, part[w][k][lane]);
        acc[k] = t;
      }
      seg_finish<NV>(p, v, col0, lane, ok, end - beg, acc);
    }
    __syncthreads();
  }
}

// Multi-CTA split of heavy targets (forward plans): a hub with thousands of incoming edges is bound by what ONE SM can
// ingest (7,278 edges x 1 KB = 7.4 MB through one CTA = 150 us on the Zipf-skewed PPI batch).  Every RGNN_HEAVY_CHUNK edges
// of a heavy segment are one work item: a CTA reduces it to a partial row in scratch (8 warps, fixed combination order),
// then one warp per heavy target adds its partial rows in item order and applies the row epilogue.  Still deterministic.
template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_reduce_heavy_part_kernel(const __grid_constant__ SegParams p) {
  __shared__ float4 part[WARPS_PER_BLOCK][NV][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col0 = blockIdx.y * (128 * NV) + lane * 4;
  const int nitems = min(*p.heavy_item_count, p.heavy_items_cap);
  bool ok[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) ok[k] = (col0 + k * 128) < p.D;
  for (int it = blockIdx.x; it < nitems; it += gridDim.x) {
    const int2 vc = __ldg(reinterpret_cast<const int2*>(p.heavy_items) + it);
    const int v = vc.x;
    if (v >= p.V) continue;                             // CTA-uniform: no __syncthreads is skipped by part of the block
    const int seg_end = __ldg(p.seg_off + v + 1);
    const int beg = __ldg(p.seg_off + v) + vc.y * p.heavy_chunk;
    const int end = min(seg_end, beg + p.heavy_chunk);
    float4 acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = f4(MAXAGG ? -FLT_MAX : 0.0f);
    seg_accumulate<NV, MODE, MAXAGG, SCALED, ACTMSG>(p, v, col0, lane, ok, beg, end, warp, WARPS_PER_BLOCK, acc);
#pragma unroll
    for (int k = 0; k < NV; ++k) part[warp][k][lane] = acc[k];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        float4 t = part[0][k][lane];
#pragma unroll
        for (int w = 1; w < WARPS_PER_BLOCK; ++w) t = MAXAGG ? max4(t, part[w][k][lane]) : add4(t, part[w][k][lane]);
        if (ok[k]) *reinterpret_cast<float4*>(p.heavy_scratch + (size_t)it * p.D + col0 + k * 128) = t;
      }
    }
    __syncthreads();
  }
}

template <int NV, bool MAXAGG>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_reduce_heavy_finish_kernel(const __grid_constant__ SegParams p) {
  const int lane = threadIdx.x & 31;
  const int col0 = blockIdx.y * (128 * NV) + lane * 4;
  const int nheavy = *p.heavy_count;
  bool ok[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) ok[k] = (col0 + k * 128) < p.D;
  for (int i = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5); i < nheavy; i += gridDim.x * WARPS_PER_BLOCK) {
    const int v = __ldg(p.heavy_list + i);
    if (v >= p.V) continue;
    const int deg = __ldg(p.seg_off + v + 1) - __ldg(p.seg_off + v);
    const int base = __ldg(p.heavy_base + i), n = (deg + p.heavy_chunk - 1) / p.heavy_chunk;
    float4 acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = f4(MAXAGG ? -FLT_MAX : 0.0f);
    for (int c = 0; c < n; ++c) {                       // fixed order: deterministic
      const float* row = p.heavy_scratch + (size_t)(base + c) * p.D + col0;
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (ok[k]) {
          const float4 t = *reinterpret_cast<const float4*>(row + k * 128);
          acc[k] = MAXAGG ? max4(acc[k], t) : add4(acc[k], t);
        }
    }
    seg_finish<NV>(p, v, col0, lane, ok, deg, acc);
  }
}

// ---- RGDCN (gnns/rgdcn.py:121-171): per-channel K x K kernels that depend on the TARGET ----------------------
// One warp per target; lane owns NV float4 of the D = C*K state (column 4*lane + 128*k), i.e. 4 outputs j0..j0+3 of
// one channel c.  The K/4 lanes of a channel are consecutive (K is a power of two <= 128), so the K inputs of the
// channel's matvec are exchanged with shuffles inside that lane group.
//   sum / mean / sqrt_n: every message of a (target, type) run shares W[v, l] and the scale, so the raw source rows
//     are summed first (one gather-add per edge, like the RGCN edge stage) and ONE K x K matvec per channel is applied
//     per run:  sum_u s (h_u[c] . W) = (s sum_u h_u[c]) . W;
//   max: the message itself is needed per edge -> matvec per edge (W rows come from L1).
template <int NV>
__device__ __forceinline__ void rgdcn_apply(const RgdcnParams& p, int v, int ty, int lane, int gbase, const bool (&ok)[NV],
                                            const float4 (&x)[NV], float scale, float4 (&m)[NV]) {
  const int K = p.K;
  const float* wrow = p.wdyn + ((size_t)v * p.L + ty) * ((size_t)p.D * K);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    m[k] = f4(0.0f);
    const int col = lane * 4 + k * 128;
    const float* wc = wrow + (size_t)(col / K) * K * K + (col % K);   // W[v, l, c, i, j0..j0+3] = wc[i * K]
    for (int q = 0; q < K / 4; ++q) {
      const float x0 = __shfl_sync(0xffffffffu, x[k].x, gbase + q), x1 = __shfl_sync(0xffffffffu, x[k].y, gbase + q);
      const float x2 = __shfl_sync(0xffffffffu, x[k].z, gbase + q), x3 = __shfl_sync(0xffffffffu, x[k].w, gbase + q);
      if (ok[k]) {
        const float4 w0 = ldg4(wc + (size_t)(4 * q) * K), w1 = ldg4(wc + (size_t)(4 * q + 1) * K);
        const float4 w2 = ldg4(wc + (size_t)(4 * q + 2) * K), w3 = ldg4(wc + (size_t)(4 * q + 3) * K);
        m[k].x = fmaf(x0, w0.x, m[k].x); m[k].y = fmaf(x0, w0.y, m[k].y); m[k].z = fmaf(x0, w0.z, m[k].z); m[k].w = fmaf(x0, w0.w, m[k].w);
        m[k].x = fmaf(x1, w1.x, m[k].x); m[k].y = fmaf(x1, w1.y, m[k].y); m[k].z = fmaf(x1, w1.z, m[k].z); m[k].w = fmaf(x1, w1.w, m[k].w);
        m[k].x = fmaf(x2, w2.x, m[k].x); m[k].y = fmaf(x2, w2.y, m[k].y); m[k].z = fmaf(x2, w2.z, m[k].z); m[k].w = fmaf(x2, w2.w, m[k].w);
        m[k].x = fmaf(x3, w3.x, m[k].x); m[k].y = fmaf(x3, w3.y, m[k].y); m[k].z = fmaf(x3, w3.z, m[k].z); m[k].w = fmaf(x3, w3.w, m[k].w);
      }
    }
    m[k] = mul4(m[k], scale);
  }
}

template <int NV, bool MAXAGG>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) rgdcn_edge_kernel(const __grid_constant__ RgdcnParams p) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  const int gbase = lane - ((lane * 4) % p.K) / 4;     // first lane of this lane's channel group (128 % K == 0)
  bool ok[NV];
  float4 acc[NV], run[NV], m[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = (lane * 4 + k * 128) < p.D;
    acc[k] = f4(MAXAGG ? -FLT_MAX : 0.0f);
    run[k] = f4(0.0f);
  }
  int cur_type = -1;
  auto scale_of = [&](int ty) { return p.num_incoming != nullptr ? 1.0f / (__ldg(p.num_incoming + (size_t)ty * p.scale_ld + v) + 1e-7f) : 1.0f; };
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) { my_src = __ldg(p.e_src + e0 + lane); my_type = __ldg(p.e_type + e0 + lane); }
    for (int j = 0; j < n; ++j) {
      const int src = __shfl_sync(0xffffffffu, my_src, j), ty = __shfl_sync(0xffffffffu, my_type, j);
      float4 r[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) r[k] = ok[k] ? ldg4(p.h + (size_t)src * p.D + lane * 4 + k * 128) : f4(0.0f);
      if (MAXAGG) {
        rgdcn_apply<NV>(p, v, ty, lane, gbase, ok, r, scale_of(ty), m);
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = max4(acc[k], m[k]);
      } else {
        if (ty != cur_type) {                            // warp-uniform: close the previous (v, type) run
          if (cur_type >= 0) {
            rgdcn_apply<NV>(p, v, cur_type, lane, gbase, ok, run, scale_of(cur_type), m);
#pragma unroll
            for (int k = 0; k < NV; ++k) { acc[k] = add4(acc[k], m[k]); run[k] = f4(0.0f); }
          }
          cur_type = ty;
        }
#pragma unroll
        for (int k = 0; k < NV; ++k) run[k] = add4(run[k], r[k]);
      }
    }
  }
  if (!MAXAGG && cur_type >= 0) {
    rgdcn_apply<NV>(p, v, cur_type, lane, gbase, ok, run, scale_of(cur_type), m);
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = add4(acc[k], m[k]);
  }
  SegParams f;
  f.D = p.D; f.agg = p.agg; f.act_out = p.act_out; f.out = p.out; f.ld_out = p.D;
  seg_finish<NV>(f, v, lane * 4, lane, ok, end - beg, acc);   // col0 carries the lane's column offset
}

// ---- RGAT: per-target, per-head online softmax fused with the weighted sum -----------------
// FUSED: the per-edge logit  a_src . T[u,l,k] + a_tgt . T[v,l,k]  (rgat.py:106-115) is computed HERE from the source row the
// warp has just gathered (4 FMAs + a butterfly over the dh/4 lanes of the head) and from the target's own row, read once per
// (target, type) run -- the separate per-node score kernel and its [V, L, K] tables are gone.  Needs dh/4 to be a power of
// two <= 32 (heads must not straddle warps); otherwise the scores come from rgat_scores_kernel as before.
__device__ __forceinline__ float dot4(float4 a, float4 b) { return (a.x * b.x + a.y * b.y) + (a.z * b.z + a.w * b.w); }

template <int NV, bool FUSED>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_rgat_kernel(const __grid_constant__ RgatParams p) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  pdl_wait();                          // T comes from the transform GEMM launched just before
  pdl_launch_dependents();
  const int dh = p.D / p.K;   // per-head width, multiple of 4 (checked on the host)
  const int lph = dh >> 2;    // lanes per head
  const int col0 = blockIdx.y * (128 * NV) + lane * 4;   // heads are independent: a warp owns a column slice

  bool ok[NV];
  int head[NV];
  float4 acc[NV], a_src[NV], a_tgt[NV];
  float mx[NV], den[NV], s_t[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int col = col0 + k * 128;
    ok[k] = col < p.D;
    head[k] = ok[k] ? col / dh : 0;
    acc[k] = f4(0.0f); a_src[k] = f4(0.0f); a_tgt[k] = f4(0.0f);
    mx[k] = -INFINITY;
    den[k] = 0.0f; s_t[k] = 0.0f;
  }
  const size_t LK = (size_t)p.L * p.K;
  int cur_type = -1;

  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) {
      my_src = __ldg(p.e_src + e0 + lane);
      my_type = __ldg(p.e_type + e0 + lane);
    }
    for (int j = 0; j < n; j += UNROLL) {
      float4 r[UNROLL][NV];
      float lg[UNROLL][NV];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (j + u < n) {
          const int src = __shfl_sync(0xffffffffu, my_src, j + u);
          const int ty = __shfl_sync(0xffffffffu, my_type, j + u);
          const float* row = p.table + ((size_t)src * p.L + ty) * p.D + col0;
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            r[u][k] = ok[k] ? ldg4(row + k * 128) : f4(0.0f);
            if (!FUSED && ok[k])
              lg[u][k] = __ldg(p.s_src + (size_t)src * LK + (size_t)ty * p.K + head[k]) + __ldg(p.s_tgt + (size_t)v * LK + (size_t)ty * p.K + head[k]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (j + u < n) {
          if (FUSED) {
            const int ty = __shfl_sync(0xffffffffu, my_type, j + u);
            if (ty != cur_type) {        // warp-uniform: new (target, type) run -> this type's attention vector, the target's score
              cur_type = ty;
              const float* trow = p.table + ((size_t)v * p.L + ty) * p.D + col0;
#pragma unroll
              for (int k = 0; k < NV; ++k) {
                float part = 0.0f;
                if (ok[k]) {
                  const float* a = p.att.att[ty] + (size_t)head[k] * 2 * dh + ((col0 + k * 128) - head[k] * dh);   // rgat.py:110-111
                  a_src[k] = ldg4(a);
                  a_tgt[k] = ldg4(a + dh);
                  part = dot4(ldg4(trow + k * 128), a_tgt[k]);
                }
                for (int o = lph >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                s_t[k] = part;
              }
            }
#pragma unroll
            for (int k = 0; k < NV; ++k) {
              float part = ok[k] ? dot4(r[u][k], a_src[k]) : 0.0f;
              for (int o = lph >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
              lg[u][k] = part + s_t[k];
            }
          }
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (ok[k]) {
              float x = lg[u][k];
              x = x > 0.0f ? x : 0.2f * x;                   // tf.nn.leaky_relu (rgat.py:113)
              if (x > mx[k]) {                                // new running maximum (rare after the first few messages): rescale
                const float corr = __expf(mx[k] - x);         // exp(-inf) = 0 on the first message
                den[k] = den[k] * corr + 1.0f;
                acc[k].x = acc[k].x * corr + r[u][k].x; acc[k].y = acc[k].y * corr + r[u][k].y;
                acc[k].z = acc[k].z * corr + r[u][k].z; acc[k].w = acc[k].w * corr + r[u][k].w;
                mx[k] = x;
              } else {                                        // one exponential per message in the common case
                const float w = __expf(x - mx[k]);
                den[k] += w;
                acc[k].x = fmaf(w, r[u][k].x, acc[k].x); acc[k].y = fmaf(w, r[u][k].y, acc[k].y);
                acc[k].z = fmaf(w, r[u][k].z, acc[k].z); acc[k].w = fmaf(w, r[u][k].w, acc[k].w);
              }
            }
        }
      }
    }
  }
  float* orow = p.out + (size_t)v * p.D + col0;
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) {
      float4 o = f4(0.0f);                                    // no incoming message -> zeros (A.7)
      if (end > beg) o = make_float4(acc[k].x / den[k], acc[k].y / den[k], acc[k].z / den[k], acc[k].w / den[k]);
      *reinterpret_cast<float4*>(orow + k * 128) = act4_cold(o, p.act_out);
    }
}

// Small batches (one PPI-shaped graph: 2,245 targets) leave the kernel above with 4,490 warps -- latency-bound at 51 us for
// 120k edges where the RGCN edge stage needs 17.5 us.  Same remedy as seg_reduce_half_kernel: a warp owns a 64-column slice and
// its two half-warps gather two DIFFERENT edges per load instruction; each half runs its own online softmax (and its own
// current-type state), the two (max, denominator, accumulator) states are merged with one xor-16 exchange at the end, in a
// fixed order.  Fused scores only (lanes per head = dh/4 in {1, 2, 4, 8, 16}: a head lies inside one half-warp's 64 columns).
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) seg_rgat_half_kernel(const __grid_constant__ RgatParams p) {
  const int lane = threadIdx.x & 31, half = lane >> 4, l16 = lane & 15;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  pdl_wait();
  pdl_launch_dependents();
  const int dh = p.D / p.K, lph = dh >> 2;
  const int col = blockIdx.y * 64 + l16 * 4;
  const bool ok = col < p.D;
  const int head = ok ? col / dh : 0;
  const unsigned hmask = half ? 0xffff0000u : 0x0000ffffu;
  float4 acc = f4(0.0f), a_src = f4(0.0f), a_tgt = f4(0.0f);
  float mx = -INFINITY, den = 0.0f, s_t = 0.0f;
  int cur_type = -1;
  const float* tcol = p.table + col;

  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) {
      my_src = __ldg(p.e_src + e0 + lane);
      my_type = __ldg(p.e_type + e0 + lane);
    }
    for (int j = 0; j < n; j += 2 * UNROLL) {
      float4 r[UNROLL];
      int ty[UNROLL];
      bool valid[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int e = j + 2 * u + half;                 // <= 31
        const int src = __shfl_sync(0xffffffffu, my_src, e);
        ty[u] = __shfl_sync(0xffffffffu, my_type, e);
        valid[u] = e < n;
        r[u] = (valid[u] && ok) ? ldg4(tcol + ((size_t)src * p.L + ty[u]) * p.D) : f4(0.0f);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (valid[u]) {                                  // uniform inside a half-warp
          if (ty[u] != cur_type) {                       // this half's new (target, type) run
            cur_type = ty[u];
            float part = 0.0f;
            if (ok) {
              const float* a = p.att.att[cur_type] + (size_t)head * 2 * dh + (col - head * dh);
              a_src = ldg4(a);
              a_tgt = ldg4(a + dh);
              part = dot4(ldg4(tcol + ((size_t)v * p.L + cur_type) * p.D), a_tgt);
            }
            for (int o = lph >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(hmask, part, o);
            s_t = part;
          }
          float part = ok ? dot4(r[u], a_src) : 0.0f;
          for (int o = lph >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(hmask, part, o);
          float x = part + s_t;
          x = x > 0.0f ? x : 0.2f * x;                   // tf.nn.leaky_relu (rgat.py:113)
          if (x > mx) {                                  // new running maximum (rare after the first few messages): rescale
            const float corr = __expf(mx - x);
            den = den * corr + 1.0f;
            acc.x = acc.x * corr + r[u].x; acc.y = acc.y * corr + r[u].y;
            acc.z = acc.z * corr + r[u].z; acc.w = acc.w * corr + r[u].w;
            mx = x;
          } else {                                       // one exponential per message in the common case
            const float w = __expf(x - mx);
            den += w;
            acc.x = fmaf(w, r[u].x, acc.x); acc.y = fmaf(w, r[u].y, acc.y);
            acc.z = fmaf(w, r[u].z, acc.z); acc.w = fmaf(w, r[u].w, acc.w);
          }
        }
      }
    }
  }
  // merge the two halves' softmax states (half 0 first: fixed order)
  const float mo = __shfl_xor_sync(0xffffffffu, mx, 16), dno = __shfl_xor_sync(0xffffffffu, den, 16);
  const float4 ao = make_float4(__shfl_xor_sync(0xffffffffu, acc.x, 16), __shfl_xor_sync(0xffffffffu, acc.y, 16),
                                __shfl_xor_sync(0xffffffffu, acc.z, 16), __shfl_xor_sync(0xffffffffu, acc.w, 16));
  if (half == 0 && ok) {
    float4 o = f4(0.0f);                                 // no incoming message -> zeros (A.7)
    if (end > beg) {
      const float m = fmaxf(mx, mo);                     // half 0 saw edge 0: mx is finite
      const float c0 = __expf(mx - m), c1 = __expf(mo - m);  // exp(-inf) = 0 when half 1 saw no edge
      const float d = den * c0 + dno * c1;
      o = make_float4((acc.x * c0 + ao.x * c1) / d, (acc.y * c0 + ao.y * c1) / d, (acc.z * c0 + ao.z * c1) / d, (acc.w * c0 + ao.w * c1) / d);
    }
    *reinterpret_cast<float4*>(p.out + (size_t)v * p.D + col) = act4_cold(o, p.act_out);
  }
}

// one thread per (node, type, head)
__global__ void rgat_scores_kernel(const float* __restrict__ table, int V, int L, int D, int K,
                                   const __grid_constant__ AttnTable att, float* __restrict__ s_src,
                                   float* __restrict__ s_tgt) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)V * L * K;
  if (i >= total) return;
  const int k = (int)(i % K);
  const int l = (int)((i / K) % L);
  const int dh = D / K;
  const float* row = table + (i / K) * (long)D + (long)k * dh;      // T[n, l, k*dh : (k+1)*dh]
  const float* a = att.att[l] + (long)k * 2 * dh;                    // [src part | tgt part] (rgat.py:110-111)
  float ss = 0.0f, st = 0.0f;
  for (int c = 0; c < dh; c += 4) {
    const float4 t = ldg4(row + c);
    const float4 as = ldg4(a + c), at = ldg4(a + dh + c);
    ss += t.x * as.x + t.y * as.y + t.z * as.z + t.w * as.w;
    st += t.x * at.x + t.y * at.y + t.z * at.z + t.w * at.w;
  }
  s_src[i] = ss;
  s_tgt[i] = st;
}

// grid = (ceil(max_type_edges / WARPS), L); one warp per edge row
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) edge_build_kernel(const __grid_constant__ EdgeBuildParams p) {
  const int lane = threadIdx.x & 31;
  const int l = blockIdx.y;
  const int i = p.type_off[l] + blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (i >= p.type_off[l + 1]) return;
  const int src = __ldg(p.o_src + i), tgt = __ldg(p.o_tgt + i);
  float* xrow = p.x + (size_t)i * p.ldx;
  const float* prow = p.p + (size_t)src * p.p_stride_node + (size_t)l * p.p_stride_type;
  if (p.concat) {
    const float* qrow = p.p + (size_t)tgt * p.p_stride_node;
    for (int c = lane * 4; c < p.D; c += 128) {
      *reinterpret_cast<float4*>(xrow + c) = ldg4(prow + c);
      *reinterpret_cast<float4*>(xrow + p.D + c) = ldg4(qrow + c);
    }
  } else {
    const float* qrow = p.q + (size_t)tgt * p.q_stride_node + (size_t)l * p.q_stride_type;
    for (int c = lane * 4; c < p.D; c += 128)
      *reinterpret_cast<float4*>(xrow + c) = act4_cold(add4(ldg4(prow + c), ldg4(qrow + c)), p.act);
  }
}

template <int NV>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) layer_norm_kernel(const float* __restrict__ x, int rows, int D,
                                                                          const float* __restrict__ gamma,
                                                                          const float* __restrict__ beta,
                                                                          float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (r >= rows) return;
  bool ok[NV];
  float4 v[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = (k * 128 + lane * 4) < D;
    v[k] = ok[k] ? ldg4(x + (size_t)r * D + k * 128 + lane * 4) : f4(0.0f);
  }
  warp_layer_norm<NV>(v, ok, D, lane, gamma, beta);
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (ok[k]) *reinterpret_cast<float4*>(out + (size_t)r * D + k * 128 + lane * 4) = v[k];
}

// ---- backward helpers ------------------------------------------------------------------------------------
__device__ __forceinline__ float act_grad_from_out(float o, int act) {
  switch (act) {
    case RGNN_ACT_TANH: return 1.0f - o * o;
    case RGNN_ACT_RELU: return o > 0.0f ? 1.0f : 0.0f;
    case RGNN_ACT_LEAKY_RELU: return o > 0.0f ? 1.0f : 0.2f;
    case RGNN_ACT_ELU: return o > 0.0f ? 1.0f : o + 1.0f;                                   // d/dx (e^x - 1) = e^x = o + 1
    case RGNN_ACT_SELU: return o > 0.0f ? 1.0507009873554805f : o + 1.0507009873554805f * 1.6732632423543772f;
    default: return 1.0f;
  }
}
__device__ __forceinline__ float gelu_grad(float x) {   // d/dx [x * Phi(x)] = Phi(x) + x * phi(x)
  return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
}

__global__ void act_backward_kernel(const float* __restrict__ grad_out, const float* __restrict__ out,
                                    const float* __restrict__ pre, int V, int D4, int act, int agg,
                                    const int32_t* __restrict__ seg_off, float* __restrict__ d_agg) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)V * D4) return;
  const int v = (int)(i / D4);
  float inv = 1.0f;
  if (agg == RGNN_AGG_MEAN || agg == RGNN_AGG_SQRT_N) {
    const float n = fmaxf((float)(__ldg(seg_off + v + 1) - __ldg(seg_off + v)), 1.0f);
    inv = 1.0f / (agg == RGNN_AGG_MEAN ? n : sqrtf(n));
  }
  const float4 g = ldg4(grad_out + i * 4);
  float4 d;
  if (act == RGNN_ACT_GELU) {
    const float4 x = ldg4(pre + i * 4);
    d = make_float4(gelu_grad(x.x), gelu_grad(x.y), gelu_grad(x.z), gelu_grad(x.w));
  } else {
    const float4 o = ldg4(out + i * 4);
    d = make_float4(act_grad_from_out(o.x, act), act_grad_from_out(o.y, act), act_grad_from_out(o.z, act), act_grad_from_out(o.w, act));
  }
  *reinterpret_cast<float4*>(d_agg + i * 4) = make_float4(g.x * d.x * inv, g.y * d.y * inv, g.z * d.z * inv, g.w * d.w * inv);
}

inline int nv_for(int D) { return (D + 127) / 128; }

}  // namespace

// Targets with more than heavy_threshold incoming edges, which the warp-per-target kernels skip.  When the plan is KNOWN to
// hold heavy targets and has scratch: the multi-CTA split (partial rows per work item, then one warp per target).  Otherwise,
// unless the plan is known to hold none, a few persistent CTAs of the one-CTA-per-target kernel walk the heavy list; with an
// unread count (deferred validation) that list is usually empty.  grid_y = number of 128*NV-column slices.
template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
static void launch_seg_heavy(const SegParams& p, unsigned grid_y, cudaStream_t stream) {
  if (p.heavy_threshold <= 0 || p.heavy_known == 0) return;
  if (p.heavy_known > 0 && p.heavy_scratch != nullptr && p.heavy_items != nullptr) {
    const unsigned ix = p.heavy_items_known > 0 ? (unsigned)(p.heavy_items_known < 1184 ? p.heavy_items_known : 1184) : 296u;
    seg_reduce_heavy_part_kernel<NV, MODE, MAXAGG, SCALED, ACTMSG><<<dim3(ix, grid_y), WARPS_PER_BLOCK * 32, 0, stream>>>(p);
    const unsigned fx = (unsigned)((p.heavy_known + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
    seg_reduce_heavy_finish_kernel<NV, MAXAGG><<<dim3(fx, grid_y), WARPS_PER_BLOCK * 32, 0, stream>>>(p);
    count_launch(2);
    return;
  }
  const unsigned gx = p.heavy_known > 0 ? (unsigned)(p.heavy_known < 4 * RGNN_WAVE_SMS ? p.heavy_known : 4 * RGNN_WAVE_SMS) : (unsigned)RGNN_WAVE_SMS;
  seg_reduce_heavy_kernel<NV, MODE, MAXAGG, SCALED, ACTMSG><<<dim3(gx, grid_y), WARPS_PER_BLOCK * 32, 0, stream>>>(p);
  count_launch();
}
template <int NV, int MODE, bool MAXAGG, bool SCALED, bool ACTMSG>
static void launch_seg_pair(const SegParams& p, dim3 grid, cudaStream_t stream) {
  launch_pdl(seg_reduce_kernel<NV, MODE, MAXAGG, SCALED, ACTMSG>, grid, dim3(WARPS_PER_BLOCK * 32), 0, stream, p);
  count_launch();
  launch_seg_heavy<NV, MODE, MAXAGG, SCALED, ACTMSG>(p, grid.y, stream);
}
template <bool SCALED>
static void launch_seg_half(const SegParams& p, unsigned gx, cudaStream_t stream) {
  launch_pdl(seg_reduce_half_kernel<SCALED>, dim3(gx, (p.D + 63) / 64), dim3(WARPS_PER_BLOCK * 32), 0, stream, p);
  count_launch();
  launch_seg_heavy<1, MSG_LINEAR, false, SCALED, false>(p, (p.D + 127) / 128, stream);
}
template <int NV, int MODE, bool MAXAGG, bool SCALED>
static void launch_seg_act(const SegParams& p, dim3 grid, cudaStream_t stream) {
  if (p.act_msg != RGNN_ACT_LINEAR) launch_seg_pair<NV, MODE, MAXAGG, SCALED, true>(p, grid, stream);
  else launch_seg_pair<NV, MODE, MAXAGG, SCALED, false>(p, grid, stream);
}
template <int NV, int MODE, bool MAXAGG>
static void launch_seg_scaled(const SegParams& p, dim3 grid, cudaStream_t stream) {
  if (p.num_incoming != nullptr) launch_seg_act<NV, MODE, MAXAGG, true>(p, grid, stream);
  else launch_seg_act<NV, MODE, MAXAGG, false>(p, grid, stream);
}
template <int NV, int MODE>
static void launch_seg_variant(const SegParams& p, dim3 grid, cudaStream_t stream) {
  if (p.agg == RGNN_AGG_MAX) launch_seg_scaled<NV, MODE, true>(p, grid, stream);
  else launch_seg_scaled<NV, MODE, false>(p, grid, stream);
}
template <int NV>
static void launch_seg_nv(const SegParams& p, dim3 grid, cudaStream_t stream) {
  switch (p.msg_mode) {
    case MSG_FILM: launch_seg_variant<NV, MSG_FILM>(p, grid, stream); break;
    case MSG_ADDTGT: launch_seg_variant<NV, MSG_ADDTGT>(p, grid, stream); break;
    default: launch_seg_variant<NV, MSG_LINEAR>(p, grid, stream); break;
  }
}

int launch_seg_reduce(const SegParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0, "segment reduce: state dim %d must be a positive multiple of 4", p.D);
  RGNN_REQUIRE(p.agg >= RGNN_AGG_SUM && p.agg <= RGNN_AGG_SQRT_N, "Unknown aggregation function code %d", p.agg);
  RGNN_REQUIRE((p.stride_idx % 4) == 0 && (p.stride_type % 4) == 0 && (p.ld_out % 4) == 0 && aligned16(p.table) && aligned16(p.out),
               "segment reduce: rows must be 16-byte aligned");
  if (p.V == 0) return RGNN_OK;
  const unsigned gx = (p.V + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  RGNN_REQUIRE(p.stride_type == 0 || (p.stride_idx % p.stride_type) == 0, "segment reduce: stride_idx must be a multiple of stride_type");
  if (p.ln_gamma != nullptr) {   // the layer-norm epilogue needs the whole row inside one warp
    if (p.D > RGNN_MAX_STATE_DIM) {
      set_error("segment reduce: layer-norm epilogue supports state dim <= %d, got %d", RGNN_MAX_STATE_DIM, p.D);
      return RGNN_E_UNSUPPORTED;
    }
    // Small batches: one warp per WHOLE row leaves too few warps to hide the gather latency (PPI-shaped Edge-MLP0: 2,245
    // warps, 73 us).  Reduce with one warp per 128-column slice instead and normalise the finished rows in a second, tiny
    // pass (V x D x 8 bytes; the layer-norm kernel works in place: it holds the row in registers).
    const bool ln_split = p.D > 128 && p.ld_out == p.D && (long)p.V < (long)RGNN_WAVE_SMS * 40;
    if (ln_split) {
      SegParams q = p;
      q.ln_gamma = nullptr; q.ln_beta = nullptr;
      launch_seg_nv<1>(q, dim3(gx, (p.D + 127) / 128), stream);
      RGNN_CHECK_CUDA(cudaGetLastError());
      return launch_layer_norm(p.out, p.V, p.D, p.ln_gamma, p.ln_beta, p.out, stream);
    }
    const dim3 grid(gx, 1);
    switch (nv_for(p.D)) {
      case 1: launch_seg_nv<1>(p, grid, stream); break;
      case 2: launch_seg_nv<2>(p, grid, stream); break;
      case 3: launch_seg_nv<3>(p, grid, stream); break;
      default: launch_seg_nv<4>(p, grid, stream); break;
    }
  } else {
    // One warp per 128-column slice: measured 2.2x faster than whole-row warps at D = 256 (the loop is latency-bound, more
    // independent warps win).  Small problems: twice as many warps, two edges per load instruction (seg_reduce_half_kernel).
    const long warps128 = (long)p.V * ((p.D + 127) / 128);
    const bool use_half = p.msg_mode == MSG_LINEAR && p.agg != RGNN_AGG_MAX && p.act_msg == RGNN_ACT_LINEAR && p.D >= 64 &&
                          warps128 < (long)RGNN_WAVE_SMS * 40;
    if (use_half && p.num_incoming != nullptr) launch_seg_half<true>(p, gx, stream);
    else if (use_half) launch_seg_half<false>(p, gx, stream);
    else launch_seg_nv<1>(p, dim3(gx, (p.D + 127) / 128), stream);
  }
  RGNN_CHECK_CUDA(cudaGetLastError());
  return RGNN_OK;
}

int launch_seg_rgat(const RgatParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0 && p.K >= 1 && (p.D % p.K) == 0, "rgat: state dim %d / heads %d invalid", p.D, p.K);
  if (((p.D / p.K) % 4) != 0) {
    set_error("rgat: per-head dim %d (state dim %d / %d heads) must be a multiple of 4 in this build", p.D / p.K, p.D, p.K);
    return RGNN_E_UNSUPPORTED;
  }
  if (p.V == 0) return RGNN_OK;
  // one warp per 128-column slice of a target row (heads are independent; more resident warps win here)
  const dim3 grid((p.V + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, (p.D + 127) / 128);
  const int lph = (p.D / p.K) / 4;
  // small batches: twice as many warps, two edges per load instruction (seg_rgat_half_kernel)
  if (p.s_src == nullptr && lph <= 16 && (long)p.V * ((p.D + 127) / 128) < (long)RGNN_WAVE_SMS * 40) {
    const dim3 hgrid(grid.x, (p.D + 63) / 64);
    RGNN_CHECK_CUDA(launch_pdl(seg_rgat_half_kernel, hgrid, dim3(WARPS_PER_BLOCK * 32), 0, stream, p));
  } else if (p.s_src == nullptr) RGNN_CHECK_CUDA(launch_pdl(seg_rgat_kernel<1, true>, grid, dim3(WARPS_PER_BLOCK * 32), 0, stream, p));
  else RGNN_CHECK_CUDA(launch_pdl(seg_rgat_kernel<1, false>, grid, dim3(WARPS_PER_BLOCK * 32), 0, stream, p));
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_rgdcn_edges(const RgdcnParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && p.K >= 4 && (p.K & (p.K - 1)) == 0 && p.K <= 128 && (p.D % p.K) == 0,
               "rgdcn: channel_dim %d must be a power of two in [4, 128] dividing the state dim %d", p.K, p.D);
  if (p.D > RGNN_MAX_STATE_DIM) {
    set_error("rgdcn: state dim %d > %d is not supported in this build", p.D, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  if (p.V == 0) return RGNN_OK;
  const unsigned gx = (p.V + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  const bool mx = p.agg == RGNN_AGG_MAX;
  switch (nv_for(p.D)) {
    case 1: if (mx) rgdcn_edge_kernel<1, true><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); else rgdcn_edge_kernel<1, false><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    case 2: if (mx) rgdcn_edge_kernel<2, true><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); else rgdcn_edge_kernel<2, false><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    case 3: if (mx) rgdcn_edge_kernel<3, true><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); else rgdcn_edge_kernel<3, false><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    default: if (mx) rgdcn_edge_kernel<4, true><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); else rgdcn_edge_kernel<4, false><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
  }
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_rgat_scores(const float* table, int V, int L, int D, int K, const AttnTable& att, float* s_src,
                       float* s_tgt, cudaStream_t stream) {
  const long total = (long)V * L * K;
  if (total == 0) return RGNN_OK;
  rgat_scores_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(table, V, L, D, K, att, s_src, s_tgt);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_edge_build(const EdgeBuildParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0, "edge build: width %d must be a positive multiple of 4", p.D);
  if (p.max_type_edges == 0) return RGNN_OK;
  const dim3 grid((p.max_type_edges + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, p.L);
  edge_build_kernel<<<grid, WARPS_PER_BLOCK * 32, 0, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_act_backward(const float* grad_out, const float* out, const float* pre, int V, int D, int act, int agg,
                        const int32_t* seg_off, float* d_agg, cudaStream_t stream) {
  RGNN_REQUIRE(D > 0 && (D % 4) == 0, "act backward: dim %d must be a positive multiple of 4", D);
  RGNN_REQUIRE(act != RGNN_ACT_GELU || pre != nullptr, "act backward: gelu needs the pre-activation");
  const long n = (long)V * (D / 4);
  if (n == 0) return RGNN_OK;
  act_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(grad_out, out, pre, V, D / 4, act, agg, seg_off, d_agg);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_layer_norm(const float* x, int rows, int D, const float* gamma, const float* beta, float* out,
                      cudaStream_t stream) {
  RGNN_REQUIRE(D > 0 && (D % 4) == 0, "layer norm: dim %d must be a positive multiple of 4", D);
  if (D > RGNN_MAX_STATE_DIM) {
    set_error("layer norm: dim %d > %d not supported by this build", D, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  if (rows == 0) return RGNN_OK;
  const dim3 grid((rows + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
  switch (nv_for(D)) {
    case 1: layer_norm_kernel<1><<<grid, WARPS_PER_BLOCK * 32, 0, stream>>>(x, rows, D, gamma, beta, out); break;
    case 2: layer_norm_kernel<2><<<grid, WARPS_PER_BLOCK * 32, 0, stream>>>(x, rows, D, gamma, beta, out); break;
    case 3: layer_norm_kernel<3><<<grid, WARPS_PER_BLOCK * 32, 0, stream>>>(x, rows, D, gamma, beta, out); break;
    default: layer_norm_kernel<4><<<grid, WARPS_PER_BLOCK * 32, 0, stream>>>(x, rows, D, gamma, beta, out); break;
  }
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
