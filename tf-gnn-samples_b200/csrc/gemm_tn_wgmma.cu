// gemm_tn_wgmma.cu -- C[M, N] = A^T . B with A [K, M] and B [K, N] both row-major and K LONG (K = number of
// nodes / edges): the weight-gradient contraction  dW = X^T . dY  of every dense map on the path
// (reference: TF autodiff of the tf.keras Dense kernels, models/sparse_graph_model.py:253-260).
//
// Same arithmetic as gemm_wgmma.cu (3xTF32 split accumulation on wgmma, fp32-level accuracy), different data
// movement: both operands have K as their SLOW axis, so neither can be bulk-copied into a K-major shared-memory
// image.  The producer warps load [16 k x 32 col] sub-blocks with coalesced 128-bit loads (8 lanes = 128 contiguous
// bytes of one k row), transpose 4x4 blocks in registers and store 16-byte K-chunks into the SWIZZLE_128B image.  The
// lane -> (column group, k chunk) mapping keeps every quarter-warp of a 128-bit shared store on 8 distinct 16-byte
// bank groups:  lane = l0 | c4 << 1 | gh << 3,  column group g8 = l0 + 2 gh,  row & 7 = 4 l0 + j,
// slot = (4 h + c4) ^ (4 l0 + j) = 4 (h ^ l0) + (c4 ^ j)  -> 8 distinct slots over (l0, c4).
//
// K is split over gridDim.y CTAs per output tile (about one wave of CTAs); partial tiles go to scratch and a second
// kernel sums them in a fixed order (deterministic, no atomics).
#include "gemm.cuh"
#include "tc_ptx.cuh"

namespace rgnn {

namespace {

constexpr int TN_BM = 128, TN_BN = 128, TN_BK = 32;
constexpr int TN_IMG_BYTES = 128 * 128;                   // one hi or lo image: 128 rows x 128 B
constexpr int TN_STAGE_BYTES = 4 * TN_IMG_BYTES;          // A_hi | A_lo | B_hi | B_lo
constexpr int TN_STAGES = 3;
constexpr int TN_CONSUMERS = 2;                           // consumer warpgroup w owns output rows [64 w, 64 w + 64)
constexpr int TN_GROUPS = 2, TN_GROUP_WARPS = 4, TN_GROUP_THREADS = 128;
constexpr int TN_THREADS = 128 * (TN_CONSUMERS + TN_GROUPS);
constexpr size_t TN_SMEM = 1024 + (size_t)TN_STAGES * TN_STAGE_BYTES + 128;

__device__ __forceinline__ float comp(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

struct TnParams {
  const float* A; int lda;     // [K, M]
  const float* B; int ldb;     // [K, N]
  float* part;                 // [splits][M][N]
  int M, N, K;
  int n_tiles;
  int steps_total;             // ceil(K / 32)
  int steps_per_split;
};

__global__ void __launch_bounds__(TN_THREADS, 1) gemm_tn_wgmma_kernel(const __grid_constant__ TnParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = ring + TN_STAGES * TN_STAGE_BYTES, empty0 = full0 + 8 * TN_STAGES;
  const int m0 = ((int)blockIdx.x / p.n_tiles) * TN_BM;
  const int n0 = ((int)blockIdx.x % p.n_tiles) * TN_BN;
  const int split = blockIdx.y;
  const int step0 = split * p.steps_per_split;
  const int step1 = min(step0 + p.steps_per_split, p.steps_total);
  const int nsteps = step1 - step0;                       // >= 1 by construction of the grid

  if (tid == 0) {
    for (int s = 0; s < TN_STAGES; ++s) {
      mbar_init(full0 + 8 * s, TN_GROUP_THREADS);         // every thread of the producing group arrives
      mbar_init(empty0 + 8 * s, TN_CONSUMERS);            // one elected thread per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg >= TN_CONSUMERS) {
    // =========================== transposing producers ===========================
    const int group = wg - TN_CONSUMERS;
    const int w = (tid >> 5) % TN_GROUP_WARPS;                     // 32-column group of both tiles
    const int l0 = lane & 1, c4 = (lane >> 1) & 3, gh = lane >> 3;
    const int col = 32 * w + 4 * (l0 + 2 * gh);                     // first of this thread's 4 tile columns (= image rows)
    const bool a_ok = (m0 + col) < p.M, b_ok = (n0 + col) < p.N;
    const float* a_ptr = p.A + (m0 + col);
    const float* b_ptr = p.B + (n0 + col);
    float4 v[2][2][4];                                              // [operand][k half][k within the 4-chunk]
    auto load_step = [&](int q) {
      const int kbase = (step0 + q) * TN_BK + 4 * c4;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int k = kbase + 16 * h + i;
          const bool k_ok = k < p.K;
          v[0][h][i] = (k_ok && a_ok) ? __ldg(reinterpret_cast<const float4*>(a_ptr + (size_t)k * p.lda)) : make_float4(0.f, 0.f, 0.f, 0.f);
          v[1][h][i] = (k_ok && b_ok) ? __ldg(reinterpret_cast<const float4*>(b_ptr + (size_t)k * p.ldb)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    if (group < nsteps) load_step(group);
    for (int q = group; q < nsteps; q += TN_GROUPS) {
      const int s = q % TN_STAGES, use = q / TN_STAGES;
      if (use > 0) mbar_wait(empty0 + 8 * s, (use - 1) & 1);
      const uint32_t stage = ring + (uint32_t)(s * TN_STAGE_BYTES);
#pragma unroll
      for (int op = 0; op < 2; ++op) {
        const uint32_t img_hi = stage + (uint32_t)(op * 2 * TN_IMG_BYTES), img_lo = img_hi + TN_IMG_BYTES;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int row = col + j;
            float4 hi, lo;
            split_tf32(comp(v[op][h][0], j), hi.x, lo.x); split_tf32(comp(v[op][h][1], j), hi.y, lo.y);
            split_tf32(comp(v[op][h][2], j), hi.z, lo.z); split_tf32(comp(v[op][h][3], j), hi.w, lo.w);
            const uint32_t off = (uint32_t)(row * 128 + (((4 * h + c4) ^ (row & 7)) << 4));
            sts128(img_hi + off, hi);
            sts128(img_lo + off, lo);
          }
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(full0 + 8 * s);
      if (q + TN_GROUPS < nsteps) load_step(q + TN_GROUPS);
    }
  } else {
    // =========================== consumers: wgmma, then the partial tile straight from registers ===========================
    const bool elected = (tid & 127) == 0;
    float acc[TN_BN / 2];
#pragma unroll
    for (int i = 0; i < TN_BN / 2; ++i) acc[i] = 0.0f;
    for (int q = 0; q < nsteps; ++q) {
      const int s = q % TN_STAGES;
      mbar_wait(full0 + 8 * s, (q / TN_STAGES) & 1);
      const uint32_t stage = ring + (uint32_t)(s * TN_STAGE_BYTES);
      const uint32_t a_hi = stage + (uint32_t)(wg * 64 * 128);
      const uint64_t da_hi = make_sw128_desc(a_hi), da_lo = make_sw128_desc(a_hi + TN_IMG_BYTES);
      const uint64_t db_hi = make_sw128_desc(stage + 2 * TN_IMG_BYTES), db_lo = make_sw128_desc(stage + 3 * TN_IMG_BYTES);
      fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TN_BK / 8; ++k) {
        const uint64_t adv = (uint64_t)(k * 2);
        wgmma_tf32<TN_BN>(acc, da_lo + adv, db_hi + adv, (q | k) != 0);
        wgmma_tf32<TN_BN>(acc, da_hi + adv, db_lo + adv, 1);
        wgmma_tf32<TN_BN>(acc, da_hi + adv, db_hi + adv, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();
      fence_operands(acc);
      if (q > 0 && elected) mbar_arrive(empty0 + 8 * ((q - 1) % TN_STAGES));
    }
    wgmma_wait<0>();
    fence_operands(acc);
    float* out = p.part + (size_t)split * p.M * p.N;
    const int r_first = m0 + wg * 64 + ((tid >> 5) & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < TN_BN / 8; ++j) {
      const int c = n0 + 8 * j + 2 * (lane & 3);              // even, N % 4 == 0: c + 1 is in range with c
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = r_first + 8 * i;
        if (r < p.M && c < p.N) *reinterpret_cast<float2*>(out + (size_t)r * p.N + c) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      }
    }
  }
}

// out[blk][m, j] = sum_s part[s][m, blk * block_cols + j]   (fixed order over s)
struct TnReduceParams {
  const float* part;
  int M, N, splits, block_cols;
  float* out[RGNN_MAX_EDGE_TYPES];
  int ld_out;
};
__global__ void __launch_bounds__(256) gemm_tn_reduce_kernel(const __grid_constant__ TnReduceParams p) {
  const long i4 = (long)blockIdx.x * blockDim.x + threadIdx.x;      // float4 index in [M, N]
  const long total4 = (long)p.M * p.N / 4;
  if (i4 >= total4) return;
  const int m = (int)(i4 * 4 / p.N), n = (int)(i4 * 4 % p.N);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* src = reinterpret_cast<const float4*>(p.part) + i4;
  for (int s = 0; s < p.splits; ++s) {
    const float4 x = __ldg(src + (size_t)s * total4);
    acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
  }
  const int blk = n / p.block_cols, j = n - blk * p.block_cols;
  *reinterpret_cast<float4*>(p.out[blk] + (size_t)m * p.ld_out + j) = acc;
}

void tn_shape(int M, int N, int K, int& m_tiles, int& n_tiles, int& splits, int& steps_per_split) {
  m_tiles = (M + TN_BM - 1) / TN_BM;
  n_tiles = (N + TN_BN - 1) / TN_BN;
  const int steps = (K + TN_BK - 1) / TN_BK;
  int want = RGNN_WAVE_SMS / (m_tiles * n_tiles);
  if (want < 1) want = 1;
  if (want > steps) want = steps;
  steps_per_split = (steps + want - 1) / want;
  splits = (steps + steps_per_split - 1) / steps_per_split;
}

}  // namespace

size_t gemm_tn_scratch_floats(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0) return 4;
  int mt, nt, splits, sps;
  tn_shape(M, N, K, mt, nt, splits, sps);
  return (size_t)splits * M * N;
}

int launch_gemm_tn(const float* A, int lda, const float* B, int ldb, int M, int N, int K, const GemmTnOut& out,
                   float* scratch, cudaStream_t stream) {
  RGNN_REQUIRE(M > 0 && N > 0 && K >= 0 && (M % 4) == 0 && (N % 4) == 0, "gemm_tn: M, N must be positive multiples of 4 (M=%d N=%d)", M, N);
  RGNN_REQUIRE((lda % 4) == 0 && (ldb % 4) == 0 && aligned16(A) && aligned16(B), "gemm_tn: operands must keep 16-byte rows");
  RGNN_REQUIRE(out.block_cols > 0 && (out.block_cols % 4) == 0 && (N % out.block_cols) == 0 && N / out.block_cols <= RGNN_MAX_EDGE_TYPES,
               "gemm_tn: bad output column blocking");
  RGNN_REQUIRE(scratch != nullptr && aligned16(scratch), "gemm_tn: scratch is NULL / misaligned");
  TnReduceParams r;
  r.part = scratch; r.M = M; r.N = N; r.block_cols = out.block_cols; r.ld_out = out.ld;
  for (int b = 0; b < N / out.block_cols; ++b) {
    RGNN_REQUIRE(out.ptr[b] != nullptr && aligned16(out.ptr[b]), "gemm_tn: output block %d is NULL / misaligned", b);
    r.out[b] = out.ptr[b];
  }
  const unsigned rblocks = (unsigned)(((long)M * N / 4 + 255) / 256);
  if (K == 0) {   // empty contraction: zeros
    r.splits = 0;
    gemm_tn_reduce_kernel<<<rblocks, 256, 0, stream>>>(r);
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
    return RGNN_OK;
  }
  TnParams p;
  p.A = A; p.lda = lda; p.B = B; p.ldb = ldb; p.part = scratch; p.M = M; p.N = N; p.K = K;
  int mt, splits;
  tn_shape(M, N, K, mt, p.n_tiles, splits, p.steps_per_split);
  p.steps_total = (K + TN_BK - 1) / TN_BK;
  static bool attr_done[64] = {};   // per device
  int device = 0;
  cudaGetDevice(&device);
  const int dv = (device >= 0 && device < 64) ? device : 0;
  if (!attr_done[dv]) {
    RGNN_CHECK_CUDA(cudaFuncSetAttribute(gemm_tn_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TN_SMEM));
    attr_done[dv] = true;
  }
  gemm_tn_wgmma_kernel<<<dim3((unsigned)(mt * p.n_tiles), (unsigned)splits), TN_THREADS, TN_SMEM, stream>>>(p);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  r.splits = splits;
  gemm_tn_reduce_kernel<<<rblocks, 256, 0, stream>>>(r);
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
