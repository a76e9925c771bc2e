// rgin_backward.cu -- the element-wise kernels of rgnn_rgin_backward (layers.cu): the gradient TF autodiff gives for ONE
// timestep of gnns/rgin.py:103-139 with source-only messages (use_target_state_as_input = False).
//
//   Z_1 = h . [E_{0,1} | .. | E_{L-1,1}],  A_j = act(Z_j),  Z_{j+1}[:, l] = A_j[:, l] . E_{l,j+1},  P = Z_{n_e}
//   a[v] = agg_{(u -> v) in A_l} act(P[u, l])        (edge MLP None: agg h[u], no activation)
//   U_k = Y_{k-1} . K_k,  Y_k = act(U_k),  Y_0 = a;  n = Y_{n_a}  (no aggregation MLP: n = act(a));  out = LayerNorm(n)
//
// The message of edge (u -> v, l) depends on (u, l) only, so the whole edge MLP and its backward run on the V node rows and
// nothing per edge is stored.  The dense parts are wgmma GEMMs and the segment reductions the forward's kernels (layers.cu);
// these kernels do the rest, one pass each:
//   rgin_act_kernel         y = act(x)                                  (A_j, Y_k and n from the stored pre-activations)
//   rgin_act_grad_kernel    y = g act'(x) / div(v), rows >= valid zero  (every dZ_j, dU_k, and d_a before the source-side sum)
//   rgin_type_sum_kernel    d_h[u] = sum_l dQ[u, l] in l order           (edge MLP None)
// The layer-norm backward is film_ln_backward_kernel (film_backward.cu) with no divisor.  Every output element has one
// writer and every sum a fixed order: no atomics.
#include "seg.cuh"

namespace rgnn {

namespace {

__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

__global__ void rgin_act_kernel(const float* __restrict__ x, long n4, int act, float* __restrict__ y) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  st4(y + i * 4, act4_cold(ldg4(x + i * 4), act));
}

// out may be g or x (each element is read before it is written, by the same thread); g and x are not read for rows >= valid
__global__ void rgin_act_grad_kernel(const __grid_constant__ RginGradParams p) {
  const int W4 = p.width / 4;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows * W4) return;
  const long v = i / W4;
  if (v >= p.valid) { st4(p.out + i * 4, make_float4(0.0f, 0.0f, 0.0f, 0.0f)); return; }
  float4 g = *reinterpret_cast<const float4*>(p.g + i * 4);
  if (p.act != RGNN_ACT_LINEAR) {
    const float4 x = *reinterpret_cast<const float4*>(p.x + i * 4);
    g = make_float4(g.x * act_grad(x.x, p.act), g.y * act_grad(x.y, p.act), g.z * act_grad(x.z, p.act), g.w * act_grad(x.w, p.act));
  }
  if (p.agg == RGNN_AGG_MEAN || p.agg == RGNN_AGG_SQRT_N) {   // mean = sum / max(n,1), sqrt_n = sum / sqrt(max(n,1))
    const float n = fmaxf((float)(__ldg(p.seg_off + v + 1) - __ldg(p.seg_off + v)), 1.0f);
    const float inv = 1.0f / (p.agg == RGNN_AGG_MEAN ? n : sqrtf(n));
    g = make_float4(g.x * inv, g.y * inv, g.z * inv, g.w * inv);
  }
  st4(p.out + i * 4, g);
}

__global__ void rgin_type_sum_kernel(const float* __restrict__ dq, long V, int L, int D4, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V * D4) return;
  const long u = i / D4;
  const int c = (int)(i - u * D4) * 4, D = D4 * 4;
  const float* row = dq + (size_t)u * L * D + c;
  float4 s = ldg4(row);
  for (int l = 1; l < L; ++l) {
    const float4 b = ldg4(row + (size_t)l * D);
    s = make_float4(s.x + b.x, s.y + b.y, s.z + b.z, s.w + b.w);
  }
  st4(out + (size_t)u * D + c, s);
}

inline unsigned blocks_of(long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

int launch_rgin_act(const float* x, long n, int act, float* y, cudaStream_t stream) {
  RGNN_REQUIRE((n % 4) == 0, "rgin backward: 16-byte rows required");
  if (n == 0) return RGNN_OK;
  rgin_act_kernel<<<blocks_of(n / 4), 256, 0, stream>>>(x, n / 4, act, y);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_rgin_act_grad(const RginGradParams& p, cudaStream_t stream) {
  RGNN_REQUIRE(p.width > 0 && (p.width % 4) == 0, "rgin backward: width %d invalid", p.width);
  const long n = p.rows * (p.width / 4);
  if (n == 0) return RGNN_OK;
  rgin_act_grad_kernel<<<blocks_of(n), 256, 0, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

int launch_rgin_type_sum(const float* dq, int V, int L, int D, float* out, cudaStream_t stream) {
  RGNN_REQUIRE(D > 0 && (D % 4) == 0 && L >= 1, "rgin backward: type sum of width %d invalid", D);
  const long n = (long)V * (D / 4);
  if (n == 0) return RGNN_OK;
  rgin_type_sum_kernel<<<blocks_of(n), 256, 0, stream>>>(dq, V, L, D / 4, out);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
