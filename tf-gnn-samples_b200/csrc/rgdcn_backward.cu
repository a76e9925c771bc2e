// rgdcn_backward.cu -- the edge kernels of rgnn_rgdcn_backward (layers.cu): the gradient TF autodiff gives for ONE timestep
// of gnns/rgdcn.py:116-165 (sum / mean / sqrt_n).  D = C K; per target v, type l and channel c:
//
//   P[v,l,c] = x_v . F_{l,c}  (K*K),  W[v,l,c][i, j] = act(P[i K + j])       (x_v = h_v, or h_v[c] per channel)
//   S[v,l,c] = sum_{(u -> v) in A_l} h_u[c],  s_{l,v} = 1 / (cnt[l, v] + 1e-7) (or 1)
//   a[v,c] = sum_l s_{l,v} S[v,l,c] . W[v,l,c],  pre = a / div(v),  y = act(pre)
//
// Given g = dL/dy, delta = g act'(pre) / div(v) and
//   dS[v,l,c]_i = s sum_j W_ij delta_j          dP[v,l,c][i K + j] = s S_i delta_j act'(P[i K + j])
// (both zero where v has no edge of type l).  rgdcn_bwd_target_kernel computes them with one warp per target in the lane
// layout of rgdcn_edge_kernel (seg_kernels.cu): lane owns 4 consecutive columns of one channel per 128-column slice, the K/4
// lanes of a channel exchange values with shuffles.
//   pass 1  walks the incoming edges (sorted by type), sums each (v, l) run of source rows into S, stores S in the dS row
//           (the lane's own slots) and adds s S . W to a -- W read column-wise as the forward does;
//   pass 2  per type, reads the lane's S back, and reads W ROW-wise (rows i0..i0+3 of its channel, the lane's own
//           elements): dS = s W delta into the same slots, dP over P in place.  Every read of P by pass 1 precedes the
//           __syncwarp before pass 2, and in pass 2 each lane reads and writes only its own P elements.
// Rows v >= Vt of dS are zeroed: the reverse-index gather of layers.cu reads dS of every edge's target.
// rgdcn_chan_sum_kernel sums dP over the channels in channel order (tied full-state kernels).  No atomics: every output
// element has one writer and every sum a fixed order.
#include "seg.cuh"

namespace rgnn {

namespace {

constexpr int WARPS_PER_BLOCK = 8;

__device__ __forceinline__ float4 zero4() { return make_float4(0.0f, 0.0f, 0.0f, 0.0f); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// first float of W[v, l, c]
__device__ __forceinline__ size_t wblock(const RgdcnBwdParams& p, int v, int l, int c) {
  return ((size_t)v * p.L * p.C + (size_t)l * p.st_type + (size_t)c * p.st_chan) * ((size_t)p.K * p.K);
}

template <int NV>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32) rgdcn_bwd_target_kernel(const __grid_constant__ RgdcnBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
  if (v >= p.V) return;
  const int K = p.K, D = p.D, L = p.L;
  bool ok[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) ok[k] = (lane * 4 + k * 128) < D;
  float* dsrow = p.dS + (size_t)v * L * D + lane * 4;
  if (v >= p.Vt) {                                      // not a wanted target: contributes nothing to the source side
    for (int l = 0; l < L; ++l)
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (ok[k]) st4(dsrow + (size_t)l * D + k * 128, zero4());
    return;
  }
  const int beg = __ldg(p.seg_off + v), end = __ldg(p.seg_off + v + 1);
  const int gbase = lane - ((lane * 4) % K) / 4;       // first lane of this lane's channel group (128 % K == 0)
  auto scale_of = [&](int ty) { return p.num_incoming != nullptr ? 1.0f / (__ldg(p.num_incoming + (size_t)ty * p.scale_ld + v) + 1e-7f) : 1.0f; };

  // ---- pass 1: a[v] = sum_l s S[v,l] . W[v,l];  S stored in dS[v,l] ----
  float4 acc[NV], run[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) { acc[k] = zero4(); run[k] = zero4(); }
  unsigned long long present = 0ull;                    // bit l: v has an incoming edge of type l (L <= 64)
  int cur_type = -1;
  auto close_run = [&]() {
    const float s = scale_of(cur_type);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (ok[k]) st4(dsrow + (size_t)cur_type * D + k * 128, run[k]);
      const int col = lane * 4 + k * 128;
      const float* wc = p.P + wblock(p, v, cur_type, (col / K) % p.C) + (col % K);   // W[i, j0..j0+3] = act(wc[i K])
      float4 m = zero4();
      for (int q = 0; q < K / 4; ++q) {
        const float x0 = __shfl_sync(0xffffffffu, run[k].x, gbase + q), x1 = __shfl_sync(0xffffffffu, run[k].y, gbase + q);
        const float x2 = __shfl_sync(0xffffffffu, run[k].z, gbase + q), x3 = __shfl_sync(0xffffffffu, run[k].w, gbase + q);
        if (ok[k]) {
          const float4 w0 = act4(ld4(wc + (size_t)(4 * q) * K), p.act), w1 = act4(ld4(wc + (size_t)(4 * q + 1) * K), p.act);
          const float4 w2 = act4(ld4(wc + (size_t)(4 * q + 2) * K), p.act), w3 = act4(ld4(wc + (size_t)(4 * q + 3) * K), p.act);
          m.x = fmaf(x0, w0.x, m.x); m.y = fmaf(x0, w0.y, m.y); m.z = fmaf(x0, w0.z, m.z); m.w = fmaf(x0, w0.w, m.w);
          m.x = fmaf(x1, w1.x, m.x); m.y = fmaf(x1, w1.y, m.y); m.z = fmaf(x1, w1.z, m.z); m.w = fmaf(x1, w1.w, m.w);
          m.x = fmaf(x2, w2.x, m.x); m.y = fmaf(x2, w2.y, m.y); m.z = fmaf(x2, w2.z, m.z); m.w = fmaf(x2, w2.w, m.w);
          m.x = fmaf(x3, w3.x, m.x); m.y = fmaf(x3, w3.y, m.y); m.z = fmaf(x3, w3.z, m.z); m.w = fmaf(x3, w3.w, m.w);
        }
      }
      acc[k] = add4(acc[k], make_float4(m.x * s, m.y * s, m.z * s, m.w * s));
      run[k] = zero4();
    }
    present |= 1ull << cur_type;
  };
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    int my_src = 0, my_type = 0;
    if (lane < n) { my_src = __ldg(p.e_src + e0 + lane); my_type = __ldg(p.e_type + e0 + lane); }
    for (int j = 0; j < n; ++j) {
      const int src = __shfl_sync(0xffffffffu, my_src, j), ty = __shfl_sync(0xffffffffu, my_type, j);
      if (ty != cur_type) {                             // warp-uniform: close the previous (v, type) run
        if (cur_type >= 0) close_run();
        cur_type = ty;
      }
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (ok[k]) run[k] = add4(run[k], ldg4(p.h + (size_t)src * D + lane * 4 + k * 128));
    }
  }
  if (cur_type >= 0) close_run();

  // ---- delta = g act'(a / div) / div ----
  const float cnt = fmaxf((float)(end - beg), 1.0f);   // mean = sum / max(n,1), sqrt_n = sum / sqrt(max(n,1))
  const float div = p.agg == RGNN_AGG_MEAN ? cnt : p.agg == RGNN_AGG_SQRT_N ? sqrtf(cnt) : 1.0f;
  const float inv = 1.0f / div;
  float4 dl[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    dl[k] = zero4();
    if (ok[k]) {
      const float4 g = ldg4(p.grad_out + (size_t)v * D + lane * 4 + k * 128);
      const float4 a = make_float4(acc[k].x / div, acc[k].y / div, acc[k].z / div, acc[k].w / div);   // as seg_finish
      dl[k] = make_float4(g.x * act_grad(a.x, p.act) * inv, g.y * act_grad(a.y, p.act) * inv,
                          g.z * act_grad(a.z, p.act) * inv, g.w * act_grad(a.w, p.act) * inv);
    }
  }
  __syncwarp();

  // ---- pass 2: per type, dS = s W delta (row-wise) and dP = s S delta^T act'(P), in place ----
  for (int l = 0; l < L; ++l) {
    const bool has = (present >> l) & 1ull;
    const float s = has ? scale_of(l) : 0.0f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int col = lane * 4 + k * 128;
      float* wr = p.P + wblock(p, v, l, (col / K) % p.C) + (size_t)(col % K) * K;   // rows i0..i0+3 of W[v, l, c]
      float4 S = zero4(), ds = zero4();
      if (has && ok[k]) S = ld4(dsrow + (size_t)l * D + k * 128);
      const float c0 = s * S.x, c1 = s * S.y, c2 = s * S.z, c3 = s * S.w;
      for (int q = 0; q < K / 4; ++q) {
        const float d0 = __shfl_sync(0xffffffffu, dl[k].x, gbase + q), d1 = __shfl_sync(0xffffffffu, dl[k].y, gbase + q);
        const float d2 = __shfl_sync(0xffffffffu, dl[k].z, gbase + q), d3 = __shfl_sync(0xffffffffu, dl[k].w, gbase + q);
        if (!ok[k]) continue;
        float* w0 = wr + 4 * q;
        if (!has) {
          st4(w0, zero4()); st4(w0 + K, zero4()); st4(w0 + 2 * K, zero4()); st4(w0 + 3 * K, zero4());
          continue;
        }
        float4 pr[4] = {ld4(w0), ld4(w0 + K), ld4(w0 + 2 * K), ld4(w0 + 3 * K)};
        float dsr[4];
        const float cr[4] = {c0, c1, c2, c3};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float4 w = act4(pr[r], p.act);
          dsr[r] = fmaf(w.x, d0, fmaf(w.y, d1, fmaf(w.z, d2, w.w * d3)));
          st4(w0 + r * K, make_float4(cr[r] * d0 * act_grad(pr[r].x, p.act), cr[r] * d1 * act_grad(pr[r].y, p.act),
                                      cr[r] * d2 * act_grad(pr[r].z, p.act), cr[r] * d3 * act_grad(pr[r].w, p.act)));
        }
        ds = make_float4(ds.x + dsr[0], ds.y + dsr[1], ds.z + dsr[2], ds.w + dsr[3]);
      }
      if (ok[k]) st4(dsrow + (size_t)l * D + k * 128, make_float4(s * ds.x, s * ds.y, s * ds.z, s * ds.w));
    }
  }
}

__global__ void rgdcn_chan_sum_kernel(const float* __restrict__ dp, long rows, int C, int KK4, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;   // float4 index in out [rows, KK]
  if (i >= rows * KK4) return;
  const long r = i / KK4;
  const int j = (int)(i - r * KK4) * 4, KK = KK4 * 4;
  const float* src = dp + (size_t)r * C * KK + j;
  float4 s = ldg4(src);
  for (int c = 1; c < C; ++c) s = add4(s, ldg4(src + (size_t)c * KK));
  st4(out + (size_t)r * KK + j, s);
}

}  // namespace

int launch_rgdcn_bwd_target(const RgdcnBwdParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.K >= 4 && (p.K & (p.K - 1)) == 0 && p.K <= 128 && p.C * p.K == p.D,
               "rgdcn_backward: channel_dim %d must be a power of two in [4, 128] dividing the state dim %d", p.K, p.D);
  RGNN_REQUIRE(p.L >= 1 && p.L <= RGNN_MAX_EDGE_TYPES, "rgdcn_backward: %d edge types out of range", p.L);
  if (p.D > RGNN_MAX_STATE_DIM) {
    set_error("rgdcn_backward: state dim %d > %d is not supported in this build", p.D, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  if (p.V == 0) return RGNN_OK;
  const int nv = (p.D + 127) / 128;
  const unsigned gx = (unsigned)((p.V + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
  switch (nv) {
    case 1: rgdcn_bwd_target_kernel<1><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    case 2: rgdcn_bwd_target_kernel<2><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    case 3: rgdcn_bwd_target_kernel<3><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
    default: rgdcn_bwd_target_kernel<4><<<gx, WARPS_PER_BLOCK * 32, 0, stream>>>(p); break;
  }
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_rgdcn_chan_sum(const float* dp, long rows, int C, int KK, float* out, cudaStream_t stream) {
  RGNN_REQUIRE(C >= 1 && KK > 0 && (KK % 4) == 0, "rgdcn_backward: channel sum of %d x %d invalid", C, KK);
  const long n = rows * (KK / 4);
  if (n == 0) return RGNN_OK;
  rgdcn_chan_sum_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dp, rows, C, KK / 4, out);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
