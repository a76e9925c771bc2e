// gemm.cuh -- node-level dense contraction on the tensor cores, fp32-accurate (3xTF32 split).
#pragma once
#include "common.cuh"

namespace rgnn {

enum GemmEpilogue {
  EPI_STORE = 0,    // C = act(acc + bias)
  EPI_GRU_ZR = 1,   // N = 2d: g = hard_sigmoid(acc + bias); cols [0,d): Z = g ; cols [d,2d): RH = g * h
  EPI_GRU_OUT = 2,  // N = d : hh = act(acc + bias); C = z*h + (1-z)*hh
};

enum GemmBatchMode {
  BATCH_NONE = 0,
  BATCH_SHARED_A = 1,   // z = type: A shared, B = bptr[z], C columns offset z * N            (T = H . [W_0|..|W_{L-1}])
  BATCH_ROW_RANGES = 2, // z = type: rows [row_off[z], row_off[z+1]) of A and C, B = bptr[z]   (per-edge MLP layers)
  BATCH_COL_BLOCKS = 3, // z = type: A columns offset z * K, B = bptr[z], C columns offset z * N (per-node MLP chains)
  BATCH_K_BLOCKS_T = 4, // one GEMM with K = batch * k_block: B[(z, j), n] = bptr[z][n * ldb1 + j]  (d_H = d_T . [W_0|..|W_{L-1}]^T)
};

struct GemmParams {
  // A = [A1 | A2] along K (A2 optional, K2 = 0 when absent); B = [B1 ; B2] along K
  const float* A1 = nullptr; int lda1 = 0; int K1 = 0;
  const float* A2 = nullptr; int lda2 = 0; int K2 = 0;
  const float* B1 = nullptr; int ldb1 = 0;
  const float* B2 = nullptr; int ldb2 = 0;
  float* C = nullptr; int ldc = 0;
  int M = 0, N = 0;
  const float* bias = nullptr;
  int epi = EPI_STORE;
  int act = RGNN_ACT_LINEAR;
  // epilogue operands (GRU): h [M, d] and z [M, d]; second output RH [M, d]
  const float* aux_h = nullptr; int ld_h = 0;
  const float* aux_z = nullptr; int ld_z = 0;
  float* C2 = nullptr; int ldc2 = 0;
  // batching over blockIdx.z
  int batch_mode = BATCH_NONE;
  int batch = 1;
  const float* bptr[RGNN_MAX_EDGE_TYPES];     // per-batch B1 (row offset for B2-style splits handled by caller)
  const float* bptr2[RGNN_MAX_EDGE_TYPES];    // per-batch B2 (optional)
  int row_off[RGNN_MAX_EDGE_TYPES + 1];       // BATCH_ROW_RANGES
  int max_rows = 0;                           // max rows of any batch entry (grid sizing)
  int k_block = 0;                            // BATCH_K_BLOCKS_T: rows of K contributed by each bptr[z] (its column count)
  const int32_t* a_rows = nullptr;            // gathered A: output row r reads A1 row a_rows[r] (compact (source, type) transform)
};

// Hopper path (gemm_wgmma.cu): wgmma tf32 with register accumulators.  Needs scratch for
// the pre-swizzled hi/lo weight images (gemm_tc_pack_bytes).  The scratch may be reused as soon as the call
// returns as long as later users are ordered on the same stream.
size_t gemm_tc_pack_bytes(const GemmParams& p);
size_t gemm_tc_pack_bytes_uncached(const GemmParams& p);   // what a call needs when the weight-image cache is off
int launch_gemm_tc(const GemmParams& p, void* pack_ws, size_t pack_ws_bytes, cudaStream_t stream);

// Optional cache of the packed weight images (static weights).  See rgnn_set_weight_cache in include/rgnn.h.
void gemm_weight_cache_enable(bool on);
void gemm_weight_cache_clear();
bool gemm_weight_cache_enabled();

// C[M, N] = A^T . B, A [K, M] (lda), B [K, N] (ldb), K long (gemm_tn_wgmma.cu): split-K over one wave of CTAs,
// deterministic two-stage sum.  The result is written as N / block_cols column blocks, block b to ptr[b] (row
// stride ld) -- one block per edge type for the per-type kernels' gradients.
struct GemmTnOut {
  float* ptr[RGNN_MAX_EDGE_TYPES];
  int block_cols = 0;
  int ld = 0;
};
size_t gemm_tn_scratch_floats(int M, int N, int K);
int launch_gemm_tn(const float* A, int lda, const float* B, int ldb, int M, int N, int K, const GemmTnOut& out,
                   float* scratch, cudaStream_t stream);

}  // namespace rgnn
