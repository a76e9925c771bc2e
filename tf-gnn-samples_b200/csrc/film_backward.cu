// film_backward.cu -- the node- and edge-level kernels of rgnn_film_backward (layers.cu): the gradient TF autodiff gives for
// ONE timestep of gnns/gnn_film.py:85-120, computed from the node tables alone.
//
//   T[u,l] = h_u . W_l,  [gamma|beta][v,l] = h_v . F_l,  s = 1/(c[l,v] + 1e-7) (or 1)
//   pre_e = gamma[v,l] * (s T[u,l]) + beta[v,l],  a[v] = agg_e act(pre_e),  y = LayerNorm(a)
//
// Nothing per edge is stored: both edge kernels recompute pre_e from T, [gamma|beta] and the node-level d_a.
//   film_ln_backward_kernel      d_a = LayerNorm'(a)^T grad_out / div(v), plus per-CTA partial sums of d_ln_gamma / d_ln_beta
//   film_bwd_target_kernel       CSR by target: g_e = act'(pre_e) * d_a[v]; dFW[v,l] = [sum g_e * s T[u,l] | sum g_e] per run
//   film_bwd_source_kernel       reverse index, segment (u,l): dT[u,l] = sum s * gamma[v,l] * g_e
// Targets / (source, type) segments with more than RGNN_HEAVY_SEGMENT edges are skipped by the warp kernels and reduced by a
// whole CTA each (the *_heavy_kernel variants).  Every output element has one writer and every sum a fixed order.
#include "seg.cuh"

namespace rgnn {

namespace {

constexpr int FB_WARPS = 8;
constexpr int FB_UNROLL = 4;   // edges in flight per warp

__device__ __forceinline__ float4 z4() { return make_float4(0.0f, 0.0f, 0.0f, 0.0f); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 scl4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// g = act'(gamma * st + beta) * d_a, element-wise
__device__ __forceinline__ float4 edge_grad(float4 gm, float4 st, float4 bt, float4 da, int act) {
  return make_float4(act_grad(gm.x * st.x + bt.x, act) * da.x, act_grad(gm.y * st.y + bt.y, act) * da.y,
                     act_grad(gm.z * st.z + bt.z, act) * da.z, act_grad(gm.w * st.w + bt.w, act) * da.w);
}

__device__ __forceinline__ float scale_of(const FilmBwdParams& p, int ty, int v) {
  return p.num_incoming != nullptr ? 1.0f / (__ldg(p.num_incoming + (size_t)ty * p.scale_ld + v) + 1e-7f) : 1.0f;
}

// ---- LayerNorm backward (eps 1e-12, biased variance: tf.contrib.layers.layer_norm) ------------------------------------
// One warp per row, grid-stride over the rows with a fixed grid: d_a overwrites a in place.  Each CTA leaves its partial
// sums of grad_out * x_hat and grad_out in partial[blockIdx.x, 2D]; film_ln_param_reduce_kernel adds them in CTA order.
template <int NV>
__global__ void __launch_bounds__(FB_WARPS * 32) film_ln_backward_kernel(const __grid_constant__ FilmLnBwdParams p) {
  __shared__ float4 red[FB_WARPS][2][NV][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D = p.D;
  bool ok[NV];
  float4 gam[NV], sg[NV], sb[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = (k * 128 + lane * 4) < D;
    gam[k] = ok[k] ? ldg4(p.ln_gamma + k * 128 + lane * 4) : z4();
    sg[k] = z4(); sb[k] = z4();
  }
  for (int v = blockIdx.x * FB_WARPS + warp; v < p.rows; v += gridDim.x * FB_WARPS) {
    float4 x[NV], go[NV];
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      x[k] = ok[k] ? *reinterpret_cast<const float4*>(p.a + (size_t)v * D + k * 128 + lane * 4) : z4();
      go[k] = ok[k] ? ldg4(p.grad_out + (size_t)v * D + k * 128 + lane * 4) : z4();
      s += (x[k].x + x[k].y) + (x[k].z + x[k].w);
    }
    const float mean = warp_sum(s) / (float)D;
    float q = 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) {
        const float a = x[k].x - mean, b = x[k].y - mean, c = x[k].z - mean, d = x[k].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
      }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)D + 1e-12f);
    float m1 = 0.0f, m2 = 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) {
        x[k] = make_float4((x[k].x - mean) * rstd, (x[k].y - mean) * rstd, (x[k].z - mean) * rstd, (x[k].w - mean) * rstd);   // x_hat
        const float4 gg = mul4(go[k], gam[k]);
        m1 += (gg.x + gg.y) + (gg.z + gg.w);
        m2 += (gg.x * x[k].x + gg.y * x[k].y) + (gg.z * x[k].z + gg.w * x[k].w);
        sg[k] = add4(sg[k], mul4(go[k], x[k]));
        sb[k] = add4(sb[k], go[k]);
      }
    m1 = warp_sum(m1) / (float)D;
    m2 = warp_sum(m2) / (float)D;
    float inv = rstd;   // rstd / div(v): mean = sum / max(n,1), sqrt_n = sum / sqrt(max(n,1)) (as launch_act_backward)
    if (p.agg == RGNN_AGG_MEAN || p.agg == RGNN_AGG_SQRT_N) {
      const float n = fmaxf((float)(__ldg(p.seg_off + v + 1) - __ldg(p.seg_off + v)), 1.0f);
      inv = rstd / (p.agg == RGNN_AGG_MEAN ? n : sqrtf(n));
    }
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) {
        const float4 gg = mul4(go[k], gam[k]);
        st4(p.a + (size_t)v * D + k * 128 + lane * 4,
            make_float4(inv * (gg.x - m1 - x[k].x * m2), inv * (gg.y - m1 - x[k].y * m2),
                        inv * (gg.z - m1 - x[k].z * m2), inv * (gg.w - m1 - x[k].w * m2)));
      }
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) { red[warp][0][k][lane] = sg[k]; red[warp][1][k][lane] = sb[k]; }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float4 a = red[0][0][k][lane], b = red[0][1][k][lane];
      for (int w = 1; w < FB_WARPS; ++w) { a = add4(a, red[w][0][k][lane]); b = add4(b, red[w][1][k][lane]); }
      if (ok[k]) {
        st4(p.partial + (size_t)blockIdx.x * 2 * D + k * 128 + lane * 4, a);
        st4(p.partial + (size_t)blockIdx.x * 2 * D + D + k * 128 + lane * 4, b);
      }
    }
  }
}

__global__ void film_ln_param_reduce_kernel(const float* __restrict__ partial, int nblk, int D, float* __restrict__ d_gamma,
                                            float* __restrict__ d_beta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * D) return;
  float acc = 0.0f;
  for (int b = 0; b < nblk; ++b) acc += partial[(size_t)b * 2 * D + c];   // CTA order: deterministic
  if (c < D) { if (d_gamma != nullptr) d_gamma[c] = acc; }
  else if (d_beta != nullptr) d_beta[c - D] = acc;
}

// ---- target side: dFW[v, l] = [sum_e g_e * s T[u,l] | sum_e g_e] over the (v, l) run ------------------------------------
// One warp per (target, 128-column slice).  Incoming edges are sorted by type, so each run is contiguous; the run's sums
// live in registers and are stored once when the type changes.  Types without an incoming edge get zero rows.
__global__ void __launch_bounds__(FB_WARPS * 32) film_bwd_target_kernel(const __grid_constant__ FilmBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * FB_WARPS + (threadIdx.x >> 5);
  if (v >= p.Vt) return;
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  if (end - beg > RGNN_HEAVY_SEGMENT) return;            // film_bwd_target_heavy_kernel
  const int D = p.D, col = blockIdx.y * 128 + lane * 4;
  const bool ok = col < D;
  const float4 da = ok ? ldg4(p.d_a + (size_t)v * D + col) : z4();
  const float* fwrow = p.FW + (size_t)v * p.L * 2 * D + col;
  float* dfrow = p.dFW + (size_t)v * p.L * 2 * D + col;
  int cur = -1;
  float4 gm = z4(), bt = z4(), dg = z4(), db = z4();
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_type = 0, my_src = 0;
    float my_scale = 1.0f;
    if (lane < n) {
      my_type = __ldg(p.e_type + e0 + lane);
      my_src = __ldg(p.e_src + e0 + lane);
      my_scale = scale_of(p, my_type, v);
    }
    for (int j = 0; j < n; j += FB_UNROLL) {
      float4 r[FB_UNROLL];
#pragma unroll
      for (int u = 0; u < FB_UNROLL; ++u) {
        const int src = __shfl_sync(0xffffffffu, my_src, j + u < 32 ? j + u : 31);
        const int ty = __shfl_sync(0xffffffffu, my_type, j + u < 32 ? j + u : 31);
        r[u] = (ok && j + u < n) ? ldg4(p.T + ((size_t)src * p.L + ty) * D + col) : z4();
      }
#pragma unroll
      for (int u = 0; u < FB_UNROLL; ++u) {
        const int ty = __shfl_sync(0xffffffffu, my_type, j + u < 32 ? j + u : 31);
        const float sc = __shfl_sync(0xffffffffu, my_scale, j + u < 32 ? j + u : 31);
        if (j + u >= n) continue;                         // warp-uniform
        if (ty != cur) {                                  // warp-uniform: close the open run, zero the skipped types
          if (cur >= 0 && ok) { st4(dfrow + (size_t)cur * 2 * D, dg); st4(dfrow + (size_t)cur * 2 * D + D, db); }
          for (int z = cur + 1; z < ty; ++z)
            if (ok) { st4(dfrow + (size_t)z * 2 * D, z4()); st4(dfrow + (size_t)z * 2 * D + D, z4()); }
          cur = ty;
          gm = ok ? ldg4(fwrow + (size_t)ty * 2 * D) : z4();
          bt = ok ? ldg4(fwrow + (size_t)ty * 2 * D + D) : z4();
          dg = z4(); db = z4();
        }
        const float4 st = scl4(r[u], sc);
        const float4 g = edge_grad(gm, st, bt, da, p.act);
        dg = add4(dg, mul4(g, st));
        db = add4(db, g);
      }
    }
  }
  if (!ok) return;
  if (cur >= 0) { st4(dfrow + (size_t)cur * 2 * D, dg); st4(dfrow + (size_t)cur * 2 * D + D, db); }
  for (int z = cur + 1; z < p.L; ++z) { st4(dfrow + (size_t)z * 2 * D, z4()); st4(dfrow + (size_t)z * 2 * D + D, z4()); }
}

// Heavy targets: one CTA per target, type by type.  The run of type l is found by binary search over the type-sorted
// segment; warp w takes its 32-edge chunks w, w + 8, ...; the 8 partial sums are added in warp order.
__global__ void __launch_bounds__(FB_WARPS * 32) film_bwd_target_heavy_kernel(const __grid_constant__ FilmBwdParams p) {
  __shared__ float4 part[FB_WARPS][2][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D = p.D, col = blockIdx.y * 128 + lane * 4;
  const bool ok = col < D;
  const int nheavy = *p.heavy_count;
  for (int i = blockIdx.x; i < nheavy; i += gridDim.x) {
    const int v = __ldg(p.heavy_list + i);
    if (v >= p.Vt) continue;                              // CTA-uniform
    const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
    const float4 da = ok ? ldg4(p.d_a + (size_t)v * D + col) : z4();
    const float* fwrow = p.FW + (size_t)v * p.L * 2 * D + col;
    float* dfrow = p.dFW + (size_t)v * p.L * 2 * D + col;
    int run_beg = beg;
    for (int ty = 0; ty < p.L; ++ty) {
      int lo = run_beg, hi = end;                         // first edge of a later type
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(p.e_type + mid) <= ty) lo = mid + 1; else hi = mid;
      }
      const int run_end = lo;
      float4 dg = z4(), db = z4();
      if (run_end > run_beg) {                            // CTA-uniform
        const float4 gm = ok ? ldg4(fwrow + (size_t)ty * 2 * D) : z4();
        const float4 bt = ok ? ldg4(fwrow + (size_t)ty * 2 * D + D) : z4();
        const float sc = scale_of(p, ty, v);
        for (int e0 = run_beg + 32 * warp; e0 < run_end; e0 += 32 * FB_WARPS) {
          const int n = min(32, run_end - e0);
          const int my_src = lane < n ? __ldg(p.e_src + e0 + lane) : 0;
          for (int j = 0; j < n; j += FB_UNROLL) {
            float4 r[FB_UNROLL];
#pragma unroll
            for (int u = 0; u < FB_UNROLL; ++u) {
              const int src = __shfl_sync(0xffffffffu, my_src, j + u < 32 ? j + u : 31);
              r[u] = (ok && j + u < n) ? ldg4(p.T + ((size_t)src * p.L + ty) * D + col) : z4();
            }
#pragma unroll
            for (int u = 0; u < FB_UNROLL; ++u)
              if (j + u < n) {
                const float4 st = scl4(r[u], sc);
                const float4 g = edge_grad(gm, st, bt, da, p.act);
                dg = add4(dg, mul4(g, st));
                db = add4(db, g);
              }
          }
        }
      }
      part[warp][0][lane] = dg; part[warp][1][lane] = db;
      __syncthreads();
      if (warp == 0 && ok) {
        float4 a = part[0][0][lane], b = part[0][1][lane];
        for (int w = 1; w < FB_WARPS; ++w) { a = add4(a, part[w][0][lane]); b = add4(b, part[w][1][lane]); }
        st4(dfrow + (size_t)ty * 2 * D, a);
        st4(dfrow + (size_t)ty * 2 * D + D, b);
      }
      __syncthreads();
      run_beg = run_end;
    }
  }
}

// ---- source side: dT[u, l] = sum over the outgoing edges (u -> v) of type l of s * gamma[v,l] * g_e ------------------------
// One warp per ((source, type) segment, 128-column slice) of the reverse index; T[u,l] is loaded once per segment.  Edges
// into targets >= Vt (not wanted on a restricted plan) contribute nothing.
__device__ __forceinline__ float4 source_edges(const FilmBwdParams& p, int ty, int col, bool ok, float4 t, int beg, int end,
                                               int chunk0, int chunk_stride, int lane) {
  float4 acc = z4();
  const int D = p.D;
  for (int e0 = beg + 32 * chunk0; e0 < end; e0 += 32 * chunk_stride) {
    const int n = min(32, end - e0);
    int my_v = 0;
    float my_scale = 1.0f;
    if (lane < n) {
      my_v = __ldg(p.rev_tgt + e0 + lane);
      if (my_v < p.Vt) my_scale = scale_of(p, ty, my_v);
    }
    for (int j = 0; j < n; j += FB_UNROLL) {
      float4 gm[FB_UNROLL], bt[FB_UNROLL], da[FB_UNROLL];
      bool use[FB_UNROLL];
#pragma unroll
      for (int u = 0; u < FB_UNROLL; ++u) {
        const int v = __shfl_sync(0xffffffffu, my_v, j + u < 32 ? j + u : 31);
        use[u] = j + u < n && v < p.Vt;                   // warp-uniform
        if (use[u] && ok) {
          const float* fw = p.FW + ((size_t)v * p.L + ty) * 2 * D + col;
          gm[u] = ldg4(fw); bt[u] = ldg4(fw + D);
          da[u] = ldg4(p.d_a + (size_t)v * D + col);
        } else {
          gm[u] = z4(); bt[u] = z4(); da[u] = z4();
        }
      }
#pragma unroll
      for (int u = 0; u < FB_UNROLL; ++u) {
        const float sc = __shfl_sync(0xffffffffu, my_scale, j + u < 32 ? j + u : 31);
        if (!use[u]) continue;
        const float4 st = scl4(t, sc);
        const float4 g = edge_grad(gm[u], st, bt[u], da[u], p.act);
        acc = add4(acc, scl4(mul4(gm[u], g), sc));
      }
    }
  }
  return acc;
}

__global__ void __launch_bounds__(FB_WARPS * 32) film_bwd_source_kernel(const __grid_constant__ FilmBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * FB_WARPS + (threadIdx.x >> 5);
  if (s >= p.V * p.L) return;
  const int beg = __ldg(p.rev_off + s), end = __ldg(p.rev_off + s + 1);
  if (end - beg > RGNN_HEAVY_SEGMENT) return;            // film_bwd_source_heavy_kernel
  const int col = blockIdx.y * 128 + lane * 4;
  const bool ok = col < p.D;
  const float4 t = (ok && end > beg) ? ldg4(p.T + (size_t)s * p.D + col) : z4();
  const float4 acc = source_edges(p, s % p.L, col, ok, t, beg, end, 0, 1, lane);
  if (ok) st4(p.dT + (size_t)s * p.D + col, acc);
}

__global__ void __launch_bounds__(FB_WARPS * 32) film_bwd_source_heavy_kernel(const __grid_constant__ FilmBwdParams p) {
  __shared__ float4 part[FB_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.y * 128 + lane * 4;
  const bool ok = col < p.D;
  const int nheavy = *p.rev_heavy_count;
  for (int i = blockIdx.x; i < nheavy; i += gridDim.x) {
    const int s = __ldg(p.rev_heavy_list + i);
    const int beg = __ldg(p.rev_off + s), end = __ldg(p.rev_off + s + 1);
    const float4 t = ok ? ldg4(p.T + (size_t)s * p.D + col) : z4();
    part[warp][lane] = source_edges(p, s % p.L, col, ok, t, beg, end, warp, FB_WARPS, lane);
    __syncthreads();
    if (warp == 0 && ok) {
      float4 a = part[0][lane];
      for (int w = 1; w < FB_WARPS; ++w) a = add4(a, part[w][lane]);
      st4(p.dT + (size_t)s * p.D + col, a);
    }
    __syncthreads();
  }
}

__global__ void add_rows_kernel(float* __restrict__ y, const float* __restrict__ x, long n4) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4* yp = reinterpret_cast<float4*>(y) + i;
  *yp = add4(*yp, ldg4(x + i * 4));
}

}  // namespace

int launch_film_ln_backward(const FilmLnBwdParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0 && p.D <= RGNN_MAX_STATE_DIM, "film backward: layer-norm dim %d invalid", p.D);
  const int nblk = film_ln_blocks(p.rows);
  if (nblk == 0) return RGNN_OK;
  const dim3 grid(nblk);
  switch ((p.D + 127) / 128) {
    case 1: film_ln_backward_kernel<1><<<grid, FB_WARPS * 32, 0, stream>>>(p); break;
    case 2: film_ln_backward_kernel<2><<<grid, FB_WARPS * 32, 0, stream>>>(p); break;
    case 3: film_ln_backward_kernel<3><<<grid, FB_WARPS * 32, 0, stream>>>(p); break;
    default: film_ln_backward_kernel<4><<<grid, FB_WARPS * 32, 0, stream>>>(p); break;
  }
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_film_ln_param_reduce(const float* partial, int rows, int D, float* d_gamma, float* d_beta, cudaStream_t stream) {
  film_ln_param_reduce_kernel<<<(2 * D + 255) / 256, 256, 0, stream>>>(partial, film_ln_blocks(rows), D, d_gamma, d_beta);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_film_edge_backward(const FilmBwdParams& p, int heavy_known, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0, "film backward: state dim %d invalid", p.D);
  const unsigned gy = (unsigned)((p.D + 127) / 128);
  if (p.Vt > 0) {   // target side: dFW
    film_bwd_target_kernel<<<dim3((unsigned)((p.Vt + FB_WARPS - 1) / FB_WARPS), gy), FB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
    if (heavy_known != 0) {   // -1: count never read back (deferred plan): a persistent wave walks the device list
      const unsigned gx = heavy_known > 0 ? (unsigned)(heavy_known < 4 * RGNN_WAVE_SMS ? heavy_known : 4 * RGNN_WAVE_SMS)
                                          : (unsigned)RGNN_WAVE_SMS;
      film_bwd_target_heavy_kernel<<<dim3(gx, gy), FB_WARPS * 32, 0, stream>>>(p);
      RGNN_CHECK_CUDA(cudaGetLastError());
      count_launch();
    }
  }
  const long segs = (long)p.V * p.L;
  if (segs > 0) {   // source side: dT (the reverse index's heavy count stays on the device, as in rgnn_rgcn_backward)
    film_bwd_source_kernel<<<dim3((unsigned)((segs + FB_WARPS - 1) / FB_WARPS), gy), FB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    film_bwd_source_heavy_kernel<<<dim3((unsigned)RGNN_WAVE_SMS, gy), FB_WARPS * 32, 0, stream>>>(p);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch(2);
  }
  return RGNN_OK;
}

int launch_add_rows(float* y, const float* x, long n, cudaStream_t stream) {
  RGNN_REQUIRE((n % 4) == 0 && aligned16(y) && aligned16(x), "add rows: 16-byte rows required");
  const long n4 = n / 4;
  if (n4 == 0) return RGNN_OK;
  add_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(y, x, n4);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
