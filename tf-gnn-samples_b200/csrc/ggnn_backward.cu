// ggnn_backward.cu -- the row kernels of rgnn_ggnn_backward (layers.cu): the gradient TF autodiff gives for ONE timestep of
// gnns/ggnn.py:71-93 with the Keras TF-1.13 cells (hard_sigmoid gates, reset_after = False, gates z | r | h).
//
//   GRU:  [a_z | a_r] = m . K_zr + h . R_zr + b_zr,  z, r = hs(a_z), hs(a_r),  a_h = m . K_h + (r h) . R_h + b_h
//         h' = z h + (1 - z) act(a_h)
//   RNN:  h' = act(a),  a = m . K + h . R + b
//
// The pre-activations come from the wgmma GEMM (layers.cu); these kernels do the element-wise parts, one pass each over
// [Vt, D]:
//   ggnn_gru_rh_kernel         r h                                                   (the operand of the a_h GEMM and of dR_h)
//   ggnn_gru_bwd_pre_kernel    da_z = g (h - act(a_h)) hs'(a_z),  da_h = g (1 - z) act'(a_h),  e = g z
//   ggnn_gru_bwd_post_kernel   da_r = d(rh) h hs'(a_r),  e += d(rh) r                (d(rh) = da_h . R_h^T, a GEMM)
//   ggnn_rnn_bwd_kernel        da = g act'(a)
// plus the bias gradient as per-CTA partial column sums added in CTA order, the divisor / restricted-target fix-up of dm and
// the final d_h += e + f.  Every output element has one writer and every sum a fixed order: no atomics.
#include "seg.cuh"

namespace rgnn {

namespace {

__device__ __forceinline__ float4 z4() { return make_float4(0.0f, 0.0f, 0.0f, 0.0f); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// d hard_sigmoid(x) / dx: 0.2 inside the linear band, 0 where the clip saturates
__device__ __forceinline__ float hs_grad(float x) { return (x > -2.5f && x < 2.5f) ? 0.2f : 0.0f; }

struct GruPre { float da_z, da_h, e; };
__device__ __forceinline__ GruPre gru_pre(float g, float h, float a_z, float a_h, int act) {
  const float z = hard_sigmoid(a_z);
  const float hh = apply_act(a_h, act);
  GruPre o;
  o.da_z = g * (h - hh) * hs_grad(a_z);
  o.da_h = g * (1.0f - z) * act_grad(a_h, act);
  o.e = g * z;
  return o;
}

// rh = hs(a_r) * h over [rows, D]; a has row stride 3D, a_r at column offset D
__global__ void ggnn_gru_rh_kernel(const float* __restrict__ a, const float* __restrict__ h, int rows, int D4,
                                   float* __restrict__ rh) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)rows * D4) return;
  const long v = i / D4;
  const int c = (int)(i - v * D4) * 4, D = D4 * 4;
  const float4 ar = ldg4(a + v * 3 * D + D + c);
  const float4 x = ldg4(h + v * D + c);
  st4(rh + v * D + c, make_float4(hard_sigmoid(ar.x) * x.x, hard_sigmoid(ar.y) * x.y, hard_sigmoid(ar.z) * x.z,
                                  hard_sigmoid(ar.w) * x.w));
}

__global__ void ggnn_gru_bwd_pre_kernel(const __grid_constant__ GgnnCellBwdParams p) {
  const int D4 = p.D / 4;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)p.rows * D4) return;
  const long v = i / D4;
  const int c = (int)(i - v * D4) * 4, D = p.D;
  const float4 g = ldg4(p.grad_out + v * D + c);
  const float4 x = ldg4(p.h + v * D + c);
  const float4 az = ldg4(p.a + v * 3 * D + c);
  const float4 ah = ldg4(p.a + v * 3 * D + 2 * D + c);
  const GruPre o0 = gru_pre(g.x, x.x, az.x, ah.x, p.act), o1 = gru_pre(g.y, x.y, az.y, ah.y, p.act);
  const GruPre o2 = gru_pre(g.z, x.z, az.z, ah.z, p.act), o3 = gru_pre(g.w, x.w, az.w, ah.w, p.act);
  st4(p.da + v * 3 * D + c, make_float4(o0.da_z, o1.da_z, o2.da_z, o3.da_z));
  st4(p.da + v * 3 * D + 2 * D + c, make_float4(o0.da_h, o1.da_h, o2.da_h, o3.da_h));
  if (p.e != nullptr) st4(p.e + v * D + c, make_float4(o0.e, o1.e, o2.e, o3.e));
}

__global__ void ggnn_gru_bwd_post_kernel(const __grid_constant__ GgnnCellBwdParams p) {
  const int D4 = p.D / 4;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)p.rows * D4) return;
  const long v = i / D4;
  const int c = (int)(i - v * D4) * 4, D = p.D;
  const float4 d = ldg4(p.drh + v * D + c);
  const float4 x = ldg4(p.h + v * D + c);
  const float4 ar = ldg4(p.a + v * 3 * D + D + c);
  st4(p.da + v * 3 * D + D + c, make_float4(d.x * x.x * hs_grad(ar.x), d.y * x.y * hs_grad(ar.y), d.z * x.z * hs_grad(ar.z),
                                            d.w * x.w * hs_grad(ar.w)));
  if (p.e != nullptr) {
    float4 e = *reinterpret_cast<const float4*>(p.e + v * D + c);
    e.x += d.x * hard_sigmoid(ar.x); e.y += d.y * hard_sigmoid(ar.y);
    e.z += d.z * hard_sigmoid(ar.z); e.w += d.w * hard_sigmoid(ar.w);
    st4(p.e + v * D + c, e);
  }
}

// da = g * act'(a), in place over a allowed (p.da == p.a): each element is read before it is written, by the same thread
__global__ void ggnn_rnn_bwd_kernel(const __grid_constant__ GgnnCellBwdParams p) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)p.rows * (p.D / 4)) return;
  const float4 g = ldg4(p.grad_out + i * 4);
  const float4 a = *reinterpret_cast<const float4*>(p.a + i * 4);
  st4(p.da + i * 4, make_float4(g.x * act_grad(a.x, p.act), g.y * act_grad(a.y, p.act), g.z * act_grad(a.z, p.act),
                                g.w * act_grad(a.w, p.act)));
}

// dm rows [0, Vt): divided by div(v) (mean: max(n,1), sqrt_n: sqrt(max(n,1)), n = all incoming edges of v); rows [Vt, V)
// (targets a restricted plan does not want: no grad_out exists for them) set to zero
__global__ void ggnn_dm_finish_kernel(float* __restrict__ dm, int V, int Vt, int D4, int agg, const int32_t* __restrict__ seg_off) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)V * D4) return;
  const int v = (int)(i / D4);
  float4* p = reinterpret_cast<float4*>(dm) + i;
  if (v >= Vt) { *p = z4(); return; }
  const float n = fmaxf((float)(__ldg(seg_off + v + 1) - __ldg(seg_off + v)), 1.0f);
  const float inv = 1.0f / (agg == RGNN_AGG_MEAN ? n : sqrtf(n));
  const float4 x = *p;
  *p = make_float4(x.x * inv, x.y * inv, x.z * inv, x.w * inv);
}

// y[0:n] += e[0:n] (+ f[0:n])
__global__ void ggnn_add_cell_grad_kernel(float* __restrict__ y, const float* __restrict__ e, const float* __restrict__ f, long n4) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 s = ldg4(e + i * 4);
  if (f != nullptr) {
    const float4 b = ldg4(f + i * 4);
    s = make_float4(s.x + b.x, s.y + b.y, s.z + b.z, s.w + b.w);
  }
  float4* yp = reinterpret_cast<float4*>(y) + i;
  const float4 a = *yp;
  *yp = make_float4(a.x + s.x, a.y + s.y, a.z + s.z, a.w + s.w);
}

// Column sums of x [rows, N]: CTA (slab, b) sums rows [b * per, (b + 1) * per) of its 128 columns, 8 row phases of 32 lanes
// each, then adds the 8 phases in order into partial[b, N]; ggnn_colsum_reduce_kernel adds the CTAs' rows in CTA order.
constexpr int CS_PHASES = 8;
__global__ void __launch_bounds__(CS_PHASES * 32) ggnn_colsum_partial_kernel(const float* __restrict__ x, int rows, int N, int per,
                                                                          float* __restrict__ partial) {
  __shared__ float4 red[CS_PHASES][32];
  const int lane = threadIdx.x & 31, ph = threadIdx.x >> 5;
  const int col = blockIdx.x * 128 + lane * 4;
  const bool ok = col < N;
  const int r0 = blockIdx.y * per, r1 = min(r0 + per, rows);
  float4 acc = z4();
  if (ok)
    for (int r = r0 + ph; r < r1; r += CS_PHASES) {
      const float4 v = ldg4(x + (size_t)r * N + col);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  red[ph][lane] = acc;
  __syncthreads();
  if (ph == 0 && ok) {
    float4 s = red[0][lane];
    for (int w = 1; w < CS_PHASES; ++w) {
      const float4 v = red[w][lane];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    st4(partial + (size_t)blockIdx.y * N + col, s);
  }
}

__global__ void ggnn_colsum_reduce_kernel(const float* __restrict__ partial, int nblk, int N, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  float acc = 0.0f;
  for (int b = 0; b < nblk; ++b) acc += partial[(size_t)b * N + c];   // CTA order: deterministic
  out[c] = acc;
}

inline unsigned blocks_of(long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

int launch_ggnn_gru_rh(const float* a, const float* h, int rows, int D, float* rh, cudaStream_t stream) {
  const long n = (long)rows * (D / 4);
  if (n == 0) return RGNN_OK;
  ggnn_gru_rh_kernel<<<blocks_of(n), 256, 0, stream>>>(a, h, rows, D / 4, rh);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_ggnn_cell_backward(const GgnnCellBwdParams& p, int cell_kind, int stage, cudaStream_t stream) {
  RGNN_REQUIRE(p.D > 0 && (p.D % 4) == 0, "ggnn backward: state dim %d invalid", p.D);
  const long n = (long)p.rows * (p.D / 4);
  if (n == 0) return RGNN_OK;
  if (cell_kind == RGNN_CELL_RNN) ggnn_rnn_bwd_kernel<<<blocks_of(n), 256, 0, stream>>>(p);
  else if (stage == 0) ggnn_gru_bwd_pre_kernel<<<blocks_of(n), 256, 0, stream>>>(p);
  else ggnn_gru_bwd_post_kernel<<<blocks_of(n), 256, 0, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_ggnn_dm_finish(float* dm, int V, int Vt, int D, int agg, const int32_t* seg_off, cudaStream_t stream) {
  const bool divide = agg == RGNN_AGG_MEAN || agg == RGNN_AGG_SQRT_N;
  const int first = divide ? 0 : Vt;   // sum: only the unwanted rows change
  const long n = (long)(V - first) * (D / 4);
  if (n <= 0) return RGNN_OK;
  // offsetting the rows keeps v >= Vt for every row of a sum launch (first == Vt), so those rows are only zeroed
  ggnn_dm_finish_kernel<<<blocks_of(n), 256, 0, stream>>>(dm + (size_t)first * D, V - first, Vt - first, D / 4, agg,
                                                          seg_off + first);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_ggnn_add_cell_grad(float* y, const float* e, const float* f, long n, cudaStream_t stream) {
  RGNN_REQUIRE((n % 4) == 0, "ggnn backward: 16-byte rows required");
  if (n == 0) return RGNN_OK;
  ggnn_add_cell_grad_kernel<<<blocks_of(n / 4), 256, 0, stream>>>(y, e, f, n / 4);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_ggnn_bias_grad(const float* x, int rows, int N, float* partial, float* out, cudaStream_t stream) {
  RGNN_REQUIRE(N > 0 && (N % 4) == 0, "ggnn backward: bias width %d invalid", N);
  const int nblk = ggnn_colsum_blocks(rows);
  if (nblk > 0) {
    const int per = (rows + nblk - 1) / nblk;
    ggnn_colsum_partial_kernel<<<dim3((unsigned)((N + 127) / 128), (unsigned)nblk), CS_PHASES * 32, 0, stream>>>(x, rows, N, per, partial);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  ggnn_colsum_reduce_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(partial, nblk, N, out);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
