// rgat_backward.cu -- the node- and edge-level kernels of rgnn_rgat_backward (layers.cu): the gradient TF autodiff gives for
// ONE timestep of gnns/rgat.py:83-139, computed from node tables alone.
//
//   T[u,l] = h_u . W_l,  s_src[u,l,k] = <a_src[l,k], T[u,l,k]>,  s_tgt[v,l,k] = <a_tgt[l,k], T[v,l,k]>
//   x_e = s_src[u,l] + s_tgt[v,l],  z_e = leaky_relu(x_e, 0.2),  alpha_e = softmax of z over ALL incoming edges of v (per head)
//   o[v,k] = sum_e alpha_e,k T[u,l,k],  y = act(o)
//
// Nothing per edge is stored: both edge kernels recompute alpha_e from the score tables and the per-(target, head) softmax
// statistics.  With d_o = act'(o) grad_y, c[v,k] = <d_o[v,k], o[v,k]>, d_alpha_e = <d_o[v,k], T[u,l,k]>,
// d_x_e = alpha_e (d_alpha_e - c[v,k]) leaky_relu'(x_e):
//   rgat_bwd_target_kernel   CSR by target: softmax statistics, o, d_o, c; D_tgt[v,l,k] = sum d_x_e over the (v, l) run
//   rgat_bwd_source_kernel   reverse index, segment (u,l): dT[u,l] = sum alpha_e d_o[v] + a_src D_src[u,l] + a_tgt D_tgt[u,l]
//   rgat_att_partial_kernel  d_att_l = [sum_u D_src[u,l,k] T[u,l,k] | sum_{v<Vt} D_tgt[v,l,k] T[v,l,k]] per CTA, added in CTA order
// A warp holds a whole row (NV float4 per lane), so a head never straddles warps whatever its width.  Per-head dot products
// use a butterfly when a head is a power-of-two group of <= 32 lanes and a shared-memory segmented sum otherwise.
// Targets / (source, type) segments with more than RGNN_HEAVY_SEGMENT edges are skipped by the warp kernels and reduced by a
// whole CTA each (the *_heavy_kernel variants).  Every output element has one writer and every sum a fixed order.
#include "seg.cuh"

namespace rgnn {

namespace {

constexpr int RB_WARPS = 8;
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float4 z4() { return make_float4(0.0f, 0.0f, 0.0f, 0.0f); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 scl4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 fma4(float s, float4 a, float4 b) {   // s * a + b
  return make_float4(fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z), fmaf(s, a.w, b.w));
}
__device__ __forceinline__ float dot4(float4 a, float4 b) { return (a.x * b.x + a.y * b.y) + (a.z * b.z + a.w * b.w); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 act_grad4(float4 x, int act) {
  return make_float4(act_grad(x.x, act), act_grad(x.y, act), act_grad(x.z, act), act_grad(x.w, act));
}
__device__ __forceinline__ float lrelu(float x) { return x > 0.0f ? x : 0.2f * x; }          // tf.nn.leaky_relu (rgat.py:113)
__device__ __forceinline__ float lrelu_grad(float x) { return x > 0.0f ? 1.0f : 0.2f; }     // TF's gradient: 0.2 at x = 0

// The lane's view of a row: chunk k covers columns k * 128 + lane * 4 .. + 3 of head head[k].
template <int NV>
struct Row {
  bool ok[NV];
  int col[NV], head[NV];
  bool lead[NV];                        // this lane holds the first column of its head: it stores the per-head scalars
  int D, K, dh, lph;
  bool fast;                            // a head is a power-of-two group of <= 32 lanes inside one chunk: butterfly
  __device__ __forceinline__ Row(const RgatBwdParams& p, int lane) {
    D = p.D; K = p.K; dh = D / K; lph = dh >> 2;
    fast = lph <= 32 && (lph & (lph - 1)) == 0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      col[k] = k * 128 + lane * 4;
      ok[k] = col[k] < D;
      head[k] = ok[k] ? col[k] / dh : 0;
      lead[k] = ok[k] && col[k] == head[k] * dh;
    }
  }
};

struct HeadScratch { float part[RGNN_MAX_STATE_DIM / 4]; float sum[RGNN_MAX_STATE_DIM / 4]; };   // one per warp

// x[k] <- the sum of x over the lanes / chunks of head[k] (warp-collective: every lane calls it with the same geometry).
template <int NV>
__device__ __forceinline__ void head_sums(float (&x)[NV], const Row<NV>& r, int lane, HeadScratch& s) {
  if (r.fast) {
    for (int o = r.lph >> 1; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < NV; ++k) x[k] += __shfl_xor_sync(FULL, x[k], o);
    return;
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) s.part[k * 32 + lane] = r.ok[k] ? x[k] : 0.0f;   // float4 index of column col[k]
  __syncwarp();
  for (int h = lane; h < r.K; h += 32) {                    // head h = float4 entries [h * lph, (h + 1) * lph), in order
    float a = 0.0f;
    for (int i = 0; i < r.lph; ++i) a += s.part[h * r.lph + i];
    s.sum[h] = a;
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < NV; ++k) x[k] = r.ok[k] ? s.sum[r.head[k]] : 0.0f;
  __syncwarp();
}

// edges in flight per warp: their loads are issued before any of them is used
template <int NV>
constexpr int edges_in_flight() { return NV <= 2 ? 4 : 2; }
__device__ __forceinline__ int lane_of(int e) { return e < 32 ? e : 31; }

// T[src, ty] and the lane's logits x = s_src[src, ty] + s_tgt[v, ty] of edge (src -> v, type ty)
template <int NV>
__device__ __forceinline__ void load_edge(const RgatBwdParams& p, const Row<NV>& r, int src, int ty, int v, float4 (&t)[NV],
                                          float (&x)[NV]) {
  const size_t LK = (size_t)p.L * p.K;
  const float* trow = p.T + ((size_t)src * p.L + ty) * p.D;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    t[k] = r.ok[k] ? ldg4(trow + r.col[k]) : z4();
    x[k] = r.ok[k] ? __ldg(p.s_src + (size_t)src * LK + (size_t)ty * p.K + r.head[k]) +
                     __ldg(p.s_tgt + (size_t)v * LK + (size_t)ty * p.K + r.head[k]) : 0.0f;
  }
}

// the warp's online softmax over edges [e0, end) in 32-edge chunks e0, e0 + 32 * stride, ...: max, denominator, sum alpha T
template <int NV>
__device__ __forceinline__ void softmax_pass(const RgatBwdParams& p, const Row<NV>& r, int v, int beg, int end, int chunk0,
                                             int stride, int lane, float (&mx)[NV], float (&den)[NV], float4 (&acc)[NV]) {
  constexpr int U = edges_in_flight<NV>();
  for (int e0 = beg + 32 * chunk0; e0 < end; e0 += 32 * stride) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) { my_src = __ldg(p.e_src + e0 + lane); my_type = __ldg(p.e_type + e0 + lane); }
    for (int j = 0; j < n; j += U) {
      float4 t[U][NV];
      float x[U][NV];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int src = __shfl_sync(FULL, my_src, lane_of(j + u)), ty = __shfl_sync(FULL, my_type, lane_of(j + u));
        if (j + u < n) load_edge<NV>(p, r, src, ty, v, t[u], x[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j + u >= n) continue;                           // warp-uniform
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          if (!r.ok[k]) continue;
          const float z = lrelu(x[u][k]);
          if (z > mx[k]) {                                  // new running maximum: rescale
            const float corr = __expf(mx[k] - z);           // exp(-inf) = 0 on the first edge
            den[k] = den[k] * corr + 1.0f;
            acc[k] = add4(scl4(acc[k], corr), t[u][k]);
            mx[k] = z;
          } else {
            const float w = __expf(z - mx[k]);
            den[k] += w;
            acc[k] = fma4(w, t[u][k], acc[k]);
          }
        }
      }
    }
  }
}

// d_x of edge (src -> v, type ty) for the lane's heads, given d_alpha (already head-summed) and v's statistics
__device__ __forceinline__ float edge_dx(float x, float m, float den, float c, float dalpha, float* alpha) {
  const float a = __expf(lrelu(x) - m) / den;
  *alpha = a;
  return a * (dalpha - c) * lrelu_grad(x);
}

// The target's statistics after pass 1: o, d_o = act'(o) grad_y, c = <d_o, o> per head; d_o row and m / den / c stored.
template <int NV>
__device__ __forceinline__ void target_stats(const RgatBwdParams& p, const Row<NV>& r, int v, bool any, int lane, HeadScratch& hs,
                                             const float (&mx)[NV], const float (&den)[NV], const float4 (&acc)[NV],
                                             float4 (&d_o)[NV], float (&c)[NV]) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    float4 o = z4();                                        // no incoming edge -> o = 0 (A.7)
    if (any && r.ok[k]) o = scl4(acc[k], 1.0f / den[k]);
    d_o[k] = r.ok[k] ? mul4(act_grad4(o, p.act), ldg4(p.grad_out + (size_t)v * p.D + r.col[k])) : z4();
    c[k] = r.ok[k] ? dot4(d_o[k], o) : 0.0f;
  }
  head_sums<NV>(c, r, lane, hs);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (r.ok[k]) st4(p.d_o + (size_t)v * p.D + r.col[k], d_o[k]);
    if (r.lead[k]) {
      const size_t i = (size_t)v * p.K + r.head[k];
      p.stat_m[i] = any ? mx[k] : 0.0f;
      p.stat_den[i] = any ? den[k] : 1.0f;
      p.stat_c[i] = c[k];
    }
  }
}

// ---- target side --------------------------------------------------------------------------------------------------------
// One warp per target.  Pass 1: online softmax -> o; then d_o, c.  Pass 2: d_x per edge; D_tgt[v,l] = sum of d_x over the
// (v, l) run, stored once when the type changes.  Types without an incoming edge get zero rows.
template <int NV>
__global__ void __launch_bounds__(RB_WARPS * 32) rgat_bwd_target_kernel(const __grid_constant__ RgatBwdParams p) {
  __shared__ HeadScratch hs_all[RB_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = blockIdx.x * RB_WARPS + warp;
  if (v >= p.Vt) return;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  if (end - beg > RGNN_HEAVY_SEGMENT) return;               // rgat_bwd_target_heavy_kernel
  HeadScratch& hs = hs_all[warp];
  const Row<NV> r(p, lane);
  float mx[NV], den[NV], c[NV];
  float4 acc[NV], d_o[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) { mx[k] = -INFINITY; den[k] = 0.0f; acc[k] = z4(); }
  softmax_pass<NV>(p, r, v, beg, end, 0, 1, lane, mx, den, acc);
  target_stats<NV>(p, r, v, end > beg, lane, hs, mx, den, acc, d_o, c);

  const size_t LK = (size_t)p.L * p.K;
  float* dtrow = p.D_tgt + (size_t)v * LK;
  int cur = -1;
  float dt[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) dt[k] = 0.0f;
  constexpr int U = edges_in_flight<NV>();
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) { my_src = __ldg(p.e_src + e0 + lane); my_type = __ldg(p.e_type + e0 + lane); }
    for (int j = 0; j < n; j += U) {
      float4 t[U][NV];
      float x[U][NV];
      int tys[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int src = __shfl_sync(FULL, my_src, lane_of(j + u));
        tys[u] = __shfl_sync(FULL, my_type, lane_of(j + u));
        if (j + u < n) load_edge<NV>(p, r, src, tys[u], v, t[u], x[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j + u >= n) continue;                           // warp-uniform
        const int ty = tys[u];
        if (ty != cur) {                                    // warp-uniform: close the open run, zero the skipped types
#pragma unroll
          for (int k = 0; k < NV; ++k)
            if (r.lead[k]) {
              if (cur >= 0) dtrow[(size_t)cur * p.K + r.head[k]] = dt[k];
              for (int z = cur + 1; z < ty; ++z) dtrow[(size_t)z * p.K + r.head[k]] = 0.0f;
            }
          cur = ty;
#pragma unroll
          for (int k = 0; k < NV; ++k) dt[k] = 0.0f;
        }
        float da[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) da[k] = dot4(d_o[k], t[u][k]);
        head_sums<NV>(da, r, lane, hs);
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (r.ok[k]) {
            float a;
            dt[k] += edge_dx(x[u][k], mx[k], den[k], c[k], da[k], &a);
          }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NV; ++k)
    if (r.lead[k]) {
      if (cur >= 0) dtrow[(size_t)cur * p.K + r.head[k]] = dt[k];
      for (int z = cur + 1; z < p.L; ++z) dtrow[(size_t)z * p.K + r.head[k]] = 0.0f;
    }
}

// Heavy targets: one CTA per target.  Pass 1: warp w runs its own online softmax over the 32-edge chunks w, w + 8, ...; the
// 8 states are merged in warp order by warp 0, which also forms d_o and c.  Pass 2 goes type by type (the run of type l is
// found by binary search over the type-sorted segment); the warps' partial D_tgt sums are added in warp order.
template <int NV>
__global__ void __launch_bounds__(RB_WARPS * 32) rgat_bwd_target_heavy_kernel(const __grid_constant__ RgatBwdParams p) {
  __shared__ HeadScratch hs_all[RB_WARPS];
  __shared__ float s_mx[RB_WARPS][NV][32], s_den[RB_WARPS][NV][32];
  __shared__ float4 s_acc[RB_WARPS][NV][32];
  __shared__ float f_m[NV][32], f_den[NV][32], f_c[NV][32];
  __shared__ float4 f_do[NV][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const Row<NV> r(p, lane);
  const size_t LK = (size_t)p.L * p.K;
  const int nheavy = *p.heavy_count;
  for (int i = blockIdx.x; i < nheavy; i += gridDim.x) {
    const int v = __ldg(p.heavy_list + i);
    if (v >= p.Vt) continue;                                // CTA-uniform
    const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
    {
      float mx[NV], den[NV];
      float4 acc[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) { mx[k] = -INFINITY; den[k] = 0.0f; acc[k] = z4(); }
      softmax_pass<NV>(p, r, v, beg, end, warp, RB_WARPS, lane, mx, den, acc);
#pragma unroll
      for (int k = 0; k < NV; ++k) { s_mx[warp][k][lane] = mx[k]; s_den[warp][k][lane] = den[k]; s_acc[warp][k][lane] = acc[k]; }
    }
    __syncthreads();
    if (warp == 0) {
      float mx[NV], den[NV], c[NV];
      float4 acc[NV], d_o[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        float m = s_mx[0][k][lane];                          // warp 0 saw the first edge: finite
        for (int w = 1; w < RB_WARPS; ++w) m = fmaxf(m, s_mx[w][k][lane]);
        float d = 0.0f;
        float4 a = z4();
        for (int w = 0; w < RB_WARPS; ++w) {
          const float s = __expf(s_mx[w][k][lane] - m);      // exp(-inf) = 0 for a warp without edges
          d = fmaf(s_den[w][k][lane], s, d);
          a = fma4(s, s_acc[w][k][lane], a);
        }
        mx[k] = m; den[k] = d; acc[k] = a;
      }
      target_stats<NV>(p, r, v, true, lane, hs_all[0], mx, den, acc, d_o, c);
#pragma unroll
      for (int k = 0; k < NV; ++k) { f_m[k][lane] = mx[k]; f_den[k][lane] = den[k]; f_c[k][lane] = c[k]; f_do[k][lane] = d_o[k]; }
    }
    __syncthreads();
    float mx[NV], den[NV], c[NV];
    float4 d_o[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) { mx[k] = f_m[k][lane]; den[k] = f_den[k][lane]; c[k] = f_c[k][lane]; d_o[k] = f_do[k][lane]; }
    int run_beg = beg;
    for (int ty = 0; ty < p.L; ++ty) {
      int lo = run_beg, hi = end;                           // first edge of a later type
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(p.e_type + mid) <= ty) lo = mid + 1; else hi = mid;
      }
      const int run_end = lo;
      float dt[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) dt[k] = 0.0f;
      constexpr int U = edges_in_flight<NV>();
      for (int e0 = run_beg + 32 * warp; e0 < run_end; e0 += 32 * RB_WARPS) {
        const int n = min(32, run_end - e0);
        const int my_src = lane < n ? __ldg(p.e_src + e0 + lane) : 0;
        for (int j = 0; j < n; j += U) {
          float4 t[U][NV];
          float x[U][NV];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int src = __shfl_sync(FULL, my_src, lane_of(j + u));
            if (j + u < n) load_edge<NV>(p, r, src, ty, v, t[u], x[u]);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (j + u >= n) continue;                       // warp-uniform
            float da[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) da[k] = dot4(d_o[k], t[u][k]);
            head_sums<NV>(da, r, lane, hs_all[warp]);
#pragma unroll
            for (int k = 0; k < NV; ++k)
              if (r.ok[k]) {
                float a;
                dt[k] += edge_dx(x[u][k], mx[k], den[k], c[k], da[k], &a);
              }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < NV; ++k) s_mx[warp][k][lane] = dt[k];
      __syncthreads();
      if (warp == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (r.lead[k]) {
            float a = s_mx[0][k][lane];
            for (int w = 1; w < RB_WARPS; ++w) a += s_mx[w][k][lane];
            p.D_tgt[(size_t)v * LK + (size_t)ty * p.K + r.head[k]] = a;
          }
      }
      __syncthreads();
      run_beg = run_end;
    }
  }
}

// ---- source side: dT[u,l] and D_src[u,l] over the outgoing edges (u -> v) of type l --------------------------------------
// T[u,l], a_src / a_tgt and s_src[u,l] are loaded once per segment.  Edges into targets >= Vt (not wanted on a restricted
// plan) contribute nothing.
template <int NV>
__device__ __forceinline__ void source_edges(const RgatBwdParams& p, const Row<NV>& r, int s, const float4 (&t)[NV],
                                             const float (&xs)[NV], int beg, int end, int chunk0, int stride, int lane,
                                             HeadScratch& hs, float4 (&acc)[NV], float (&dsrc)[NV]) {
  constexpr int U = edges_in_flight<NV>();
  const int ty = s % p.L;
  for (int e0 = beg + 32 * chunk0; e0 < end; e0 += 32 * stride) {
    const int n = min(32, end - e0);
    const int my_v = lane < n ? __ldg(p.rev_tgt + e0 + lane) : 0;
    for (int j = 0; j < n; j += U) {
      float4 d_o[U][NV];
      float x[U][NV], m[U][NV], den[U][NV], c[U][NV];
      bool use[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int v = __shfl_sync(FULL, my_v, lane_of(j + u));
        use[u] = j + u < n && v < p.Vt;                     // warp-uniform
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const bool ld = use[u] && r.ok[k];
          const size_t vk = (size_t)v * p.K + r.head[k];
          d_o[u][k] = ld ? ldg4(p.d_o + (size_t)v * p.D + r.col[k]) : z4();
          x[u][k] = ld ? xs[k] + __ldg(p.s_tgt + ((size_t)v * p.L + ty) * p.K + r.head[k]) : 0.0f;
          m[u][k] = ld ? __ldg(p.stat_m + vk) : 0.0f;
          den[u][k] = ld ? __ldg(p.stat_den + vk) : 1.0f;
          c[u][k] = ld ? __ldg(p.stat_c + vk) : 0.0f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!use[u]) continue;                              // warp-uniform
        float da[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) da[k] = dot4(d_o[u][k], t[k]);
        head_sums<NV>(da, r, lane, hs);
#pragma unroll
        for (int k = 0; k < NV; ++k)
          if (r.ok[k]) {
            float a;
            dsrc[k] += edge_dx(x[u][k], m[u][k], den[u][k], c[u][k], da[k], &a);
            acc[k] = fma4(a, d_o[u][k], acc[k]);
          }
      }
    }
  }
}

template <int NV>
__device__ __forceinline__ void source_load(const RgatBwdParams& p, const Row<NV>& r, int s, float4 (&t)[NV], float (&xs)[NV]) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    t[k] = r.ok[k] ? ldg4(p.T + (size_t)s * p.D + r.col[k]) : z4();
    xs[k] = r.ok[k] ? __ldg(p.s_src + (size_t)s * p.K + r.head[k]) : 0.0f;
  }
}

// dT[u,l] = acc + a_src D_src[u,l] + (u < Vt: a_tgt D_tgt[u,l]); D_src stored by the head's first lane
template <int NV>
__device__ __forceinline__ void source_finish(const RgatBwdParams& p, const Row<NV>& r, int s, const float4 (&acc)[NV],
                                              const float (&dsrc)[NV]) {
  const int u = s / p.L, ty = s % p.L;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!r.ok[k]) continue;
    const float* a = p.att.att[ty] + (size_t)r.head[k] * 2 * r.dh + (r.col[k] - r.head[k] * r.dh);   // rgat.py:110-111
    float4 g = fma4(dsrc[k], ldg4(a), acc[k]);
    if (u < p.Vt) g = fma4(__ldg(p.D_tgt + (size_t)s * p.K + r.head[k]), ldg4(a + r.dh), g);
    st4(p.dT + (size_t)s * p.D + r.col[k], g);
    if (r.lead[k]) p.D_src[(size_t)s * p.K + r.head[k]] = dsrc[k];
  }
}

template <int NV>
__global__ void __launch_bounds__(RB_WARPS * 32) rgat_bwd_source_kernel(const __grid_constant__ RgatBwdParams p) {
  __shared__ HeadScratch hs_all[RB_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s = blockIdx.x * RB_WARPS + warp;
  if (s >= p.V * p.L) return;
  const int beg = __ldg(p.rev_off + s), end = __ldg(p.rev_off + s + 1);
  if (end - beg > RGNN_HEAVY_SEGMENT) return;               // rgat_bwd_source_heavy_kernel
  const Row<NV> r(p, lane);
  float4 t[NV], acc[NV];
  float xs[NV], dsrc[NV];
  source_load<NV>(p, r, s, t, xs);
#pragma unroll
  for (int k = 0; k < NV; ++k) { acc[k] = z4(); dsrc[k] = 0.0f; }
  source_edges<NV>(p, r, s, t, xs, beg, end, 0, 1, lane, hs_all[warp], acc, dsrc);
  source_finish<NV>(p, r, s, acc, dsrc);
}

template <int NV>
__global__ void __launch_bounds__(RB_WARPS * 32) rgat_bwd_source_heavy_kernel(const __grid_constant__ RgatBwdParams p) {
  __shared__ HeadScratch hs_all[RB_WARPS];
  __shared__ float4 s_acc[RB_WARPS][NV][32];
  __shared__ float s_ds[RB_WARPS][NV][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const Row<NV> r(p, lane);
  const int nheavy = *p.rev_heavy_count;
  for (int i = blockIdx.x; i < nheavy; i += gridDim.x) {
    const int s = __ldg(p.rev_heavy_list + i);
    const int beg = __ldg(p.rev_off + s), end = __ldg(p.rev_off + s + 1);
    float4 t[NV], acc[NV];
    float xs[NV], dsrc[NV];
    source_load<NV>(p, r, s, t, xs);
#pragma unroll
    for (int k = 0; k < NV; ++k) { acc[k] = z4(); dsrc[k] = 0.0f; }
    source_edges<NV>(p, r, s, t, xs, beg, end, warp, RB_WARPS, lane, hs_all[warp], acc, dsrc);
#pragma unroll
    for (int k = 0; k < NV; ++k) { s_acc[warp][k][lane] = acc[k]; s_ds[warp][k][lane] = dsrc[k]; }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        float4 a = s_acc[0][k][lane];
        float d = s_ds[0][k][lane];
        for (int w = 1; w < RB_WARPS; ++w) { a = add4(a, s_acc[w][k][lane]); d += s_ds[w][k][lane]; }
        acc[k] = a; dsrc[k] = d;
      }
      source_finish<NV>(p, r, s, acc, dsrc);
    }
    __syncthreads();
  }
}

// ---- attention gradients -----------------------------------------------------------------------------------------------
// CTA (b, l) covers rows [b * rows, (b + 1) * rows); thread c owns columns 4c .. 4c + 3 (head h): its partial sums of
// D_src[u,l,h] T[u,l] and D_tgt[v,l,h] T[v,l] (v < Vt) go to partial[b, l] at the attention vector's layout.
__global__ void __launch_bounds__(RGNN_MAX_STATE_DIM / 4) rgat_att_partial_kernel(const __grid_constant__ RgatBwdParams p,
                                                                                 int rows, float* __restrict__ partial) {
  const int col = threadIdx.x * 4, l = blockIdx.y;
  if (col >= p.D) return;
  const int dh = p.D / p.K, h = col / dh;
  const int r0 = blockIdx.x * rows, r1 = min(r0 + rows, p.V);
  float4 as = z4(), at = z4();
  for (int u = r0; u < r1; ++u) {
    const size_t s = (size_t)u * p.L + l;
    const float4 t = ldg4(p.T + s * p.D + col);
    as = fma4(__ldg(p.D_src + s * p.K + h), t, as);
    if (u < p.Vt) at = fma4(__ldg(p.D_tgt + s * p.K + h), t, at);
  }
  float* out = partial + ((size_t)blockIdx.x * p.L + l) * 2 * p.D + (size_t)h * 2 * dh + (col - h * dh);
  st4(out, as);
  st4(out + dh, at);
}

__global__ void rgat_att_reduce_kernel(const float* __restrict__ partial, int nblk, int L, int D, const __grid_constant__ RgatAttOut out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * 2 * D) return;
  float acc = 0.0f;
  for (int b = 0; b < nblk; ++b) acc += partial[(size_t)b * L * 2 * D + i];   // CTA order: deterministic
  out.ptr[i / (2 * D)][i % (2 * D)] = acc;
}

template <int NV>
int launch_edges_nv(const RgatBwdParams& p, int heavy_known, cudaStream_t stream) {
  if (p.Vt > 0) {
    rgat_bwd_target_kernel<NV><<<(unsigned)((p.Vt + RB_WARPS - 1) / RB_WARPS), RB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
    if (heavy_known != 0) {   // -1: count never read back (deferred plan): a persistent wave walks the device list
      const unsigned gx = heavy_known > 0 ? (unsigned)(heavy_known < 4 * RGNN_WAVE_SMS ? heavy_known : 4 * RGNN_WAVE_SMS)
                                          : (unsigned)RGNN_WAVE_SMS;
      rgat_bwd_target_heavy_kernel<NV><<<gx, RB_WARPS * 32, 0, stream>>>(p);
      RGNN_CHECK_CUDA(cudaGetLastError());
      count_launch();
    }
  }
  const long segs = (long)p.V * p.L;
  if (segs > 0) {   // the reverse index's heavy count stays on the device, as in rgnn_rgcn_backward
    rgat_bwd_source_kernel<NV><<<(unsigned)((segs + RB_WARPS - 1) / RB_WARPS), RB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    rgat_bwd_source_heavy_kernel<NV><<<(unsigned)RGNN_WAVE_SMS, RB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch(2);
  }
  return RGNN_OK;
}

}  // namespace

int launch_rgat_edge_backward(const RgatBwdParams& p, int heavy_known, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0 && p.D <= RGNN_MAX_STATE_DIM && p.K >= 1 && (p.D % p.K) == 0 && ((p.D / p.K) % 4) == 0,
               "rgat backward: state dim %d / heads %d invalid", p.D, p.K);
  switch ((p.D + 127) / 128) {
    case 1: return launch_edges_nv<1>(p, heavy_known, stream);
    case 2: return launch_edges_nv<2>(p, heavy_known, stream);
    case 3: return launch_edges_nv<3>(p, heavy_known, stream);
    default: return launch_edges_nv<4>(p, heavy_known, stream);
  }
}

int launch_rgat_att_backward(const RgatBwdParams& p, float* partial, const RgatAttOut& out, cudaStream_t stream) {
  const int nblk = rgat_att_blocks(p.V);
  if (nblk > 0) {
    const int rows = (p.V + nblk - 1) / nblk;
    rgat_att_partial_kernel<<<dim3((unsigned)nblk, (unsigned)p.L), RGNN_MAX_STATE_DIM / 4, 0, stream>>>(p, rows, partial);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  const int n = p.L * 2 * p.D;
  rgat_att_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(partial, nblk, p.L, p.D, out);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
