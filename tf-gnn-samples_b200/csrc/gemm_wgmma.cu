// gemm_wgmma.cu -- C = epilogue([A1|A2] . [B1;B2]) on the Hopper tensor cores (wgmma, sm_90a).
//
// Contract: fp32 in / fp32 out, fp32-level accuracy through 3xTF32 split accumulation: every product is
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with hi = the TF32 part of x and lo = x - hi.
//
//   * tile: 128 rows x BN columns, BN in {32, 64, 128} chosen per problem so that the persistent grid is about one
//     wave; two consumer warpgroups hold the 64 x BN fp32 accumulators of their halves in registers;
//   * operands: K-major SWIZZLE_128B shared-memory images, one 128-byte row = 32 fp32 of K;
//       B (weights): split into TF32 hi/lo and pre-swizzled ONCE per call by pack_b_kernel into the exact
//         shared-memory image, then streamed with 1-D bulk copies (cp.async.bulk) that complete on the stage's mbarrier;
//       A (node states): two producer warpgroups take K chunks in turn, load rows with coalesced 128-bit loads,
//         split hi/lo in registers and store both images swizzled (conflict-free), then fence.proxy.async + arrive;
//   * MMA: per 32-wide K chunk, 4 k-steps x {lo*hi, hi*lo, hi*hi} wgmma.m64nBNk8.tf32 per consumer warpgroup; a stage
//     is released as soon as the wgmma group that read it has retired (wait_group 1);
//   * epilogue: straight from the accumulator registers (bias / activation / GRU gate math), while the producers
//     already fill the ring with the next tile's chunks.
#include "gemm.cuh"
#include "tc_ptx.cuh"

#include <stdlib.h>
#include <vector>
#include <mutex>
#include <algorithm>

namespace rgnn {

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;                    // fp32 elements per 128-byte swizzle row
constexpr int TC_GROUPS = 2;                 // producer warpgroups, taking K chunks round-robin (see the producer loop)
constexpr int TC_GROUP_THREADS = 128;
constexpr int TC_CONSUMERS = 2;              // consumer warpgroup w owns rows [64 w, 64 w + 64) of the tile
constexpr int TC_THREADS = 128 * (TC_CONSUMERS + TC_GROUPS);
constexpr int A_IMG_BYTES = TC_BM * 128;     // 16 KB
constexpr int A_HALF_BYTES = 64 * 128;       // one consumer's 64 rows of an A image
constexpr size_t TC_SMEM_MAX = 227 * 1024;   // opt-in dynamic shared memory per CTA on sm_90
constexpr size_t TC_RING_BUDGET = TC_SMEM_MAX - 1024 /*align*/ - 256 /*barriers*/;

// -------------------------------------------------------------------------------------------------
// pack_b: [K, N] fp32 weights -> per (n-tile, k-chunk) hi / lo shared-memory images (BN rows x 128 B,
// K-major, 128-byte swizzled).  Column blocks may come from different matrices (per-type kernels).
// -------------------------------------------------------------------------------------------------
struct PackParams {
  const float* b1[RGNN_MAX_EDGE_TYPES];   // column block j of segment 1: rows [0, K1)
  const float* b2[RGNN_MAX_EDGE_TYPES];   // column block j of segment 2: rows [0, K2) (may be null when K2 == 0)
  int ldb1, ldb2;
  int K1, K2;
  int block_cols;                         // width of one column block (N for a plain GEMM)
  int n_total;                            // total columns = blocks * block_cols
  int BN;
  int chunks1, chunks2;                   // ceil(K1/32), ceil(K2/32)
  int transposed, k_block;                // transposed: B[(z, j), n] = b1[z][n * ldb1 + j], K = blocks * k_block
  float* out;                             // [n_tiles][chunks1+chunks2][2][BN*32]
};

// grid = (k-chunks, n-tiles, BN/32 row slices... ceil), block = 256 threads = 32 image rows x 8 16-byte chunks
__global__ void __launch_bounds__(256) pack_b_kernel(const __grid_constant__ PackParams p) {
  // Programmatic dependent launch: the image buffer may still be read by the GEMM enqueued before (the layers reuse one scratch
  // region), so nothing is written before the predecessor has completed; the GEMM that consumes these images may start its
  // set-up (barrier init) right away -- it waits for this grid before touching them.
  pdl_wait();
  pdl_launch_dependents();
  const int chunk = blockIdx.x;           // k-chunk over both segments
  const int tile = blockIdx.y;            // n-tile
  const int nchunks = p.chunks1 + p.chunks2;
  const bool seg2 = chunk >= p.chunks1;
  const int k0 = (seg2 ? chunk - p.chunks1 : chunk) * TC_BK;
  const int Kseg = seg2 ? p.K2 : p.K1;
  const int ld = seg2 ? p.ldb2 : p.ldb1;
  float* img_hi = p.out + ((size_t)tile * nchunks + chunk) * 2 * (p.BN * TC_BK);
  float* img_lo = img_hi + p.BN * TC_BK;
  const int nl = blockIdx.z * 32 + (threadIdx.x & 31);   // consecutive threads -> consecutive n: coalesced reads per k
  const int c16 = threadIdx.x >> 5;                      // 16-byte chunk (4 k values) inside the 128-byte row
  if (nl >= p.BN) return;
  const int n = tile * p.BN + nl;
  float hi[4], lo[4];
  float x[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (n < p.n_total) {
    if (p.transposed) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + c16 * 4 + j;
        if (k < Kseg) {
          const int blk = k / p.k_block, jj = k - blk * p.k_block;
          x[j] = __ldg(p.b1[blk] + (size_t)n * ld + jj);
        }
      }
    } else {
      const int blk = n / p.block_cols, col = n - blk * p.block_cols;
      const float* src = (seg2 ? p.b2[blk] : p.b1[blk]) + col;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + c16 * 4 + j;
        if (k < Kseg) x[j] = __ldg(src + (size_t)k * ld);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) split_tf32(x[j], hi[j], lo[j]);
  const int off = (nl >> 3) * 256 + (nl & 7) * 32 + ((c16 ^ (nl & 7)) << 2);   // float index inside the image
  *reinterpret_cast<float4*>(img_hi + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<float4*>(img_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

struct TcParams {
  GemmParams g;
  const float* packed;     // pack_b output (per z for ROW_RANGES / COL_BLOCKS: z * packed_stride floats)
  size_t packed_stride;
  int BN, stages, chunks1, chunks2;
  int n_total;             // columns of C covered by this launch (batch*N for SHARED_A, else N)
  int n_tiles;
  int ring_bytes;
  int total_tiles;
  int tile_start[RGNN_MAX_EDGE_TYPES + 1];   // first tile of batch entry z (ROW_RANGES / COL_BLOCKS), else {0, total}
};

struct TileInfo { int z, m0, row_end, n_tile; };

__device__ __noinline__ TileInfo decode_tile(const TcParams& p, int t) {
  TileInfo ti;
  const GemmParams& g = p.g;
  int z = 0;
  if (g.batch_mode == BATCH_ROW_RANGES || g.batch_mode == BATCH_COL_BLOCKS) {
    while (t >= p.tile_start[z + 1]) ++z;
  }
  const int local = t - p.tile_start[z];
  const int row_begin = (g.batch_mode == BATCH_ROW_RANGES) ? g.row_off[z] : 0;
  ti.z = z;
  ti.row_end = (g.batch_mode == BATCH_ROW_RANGES) ? g.row_off[z + 1] : g.M;
  ti.m0 = row_begin + (local / p.n_tiles) * TC_BM;
  ti.n_tile = local % p.n_tiles;
  return ti;
}

// One consumer warpgroup's 64 x BN accumulator -> bias / activation / gate math -> C.  Each thread holds two rows and
// BN / 4 column pairs (fragment layout: tc_ptx.cuh, wgmma_tf32).
template <int EPI, int BN>
__device__ __forceinline__ void epilogue_regs(const TcParams& p, const TileInfo& ti, const float (&acc)[BN / 2], int row0, int lane) {
  const GemmParams& g = p.g;
  const int dgru = (EPI == EPI_GRU_ZR) ? g.N / 2 : g.N;
  float* C = g.C + (g.batch_mode == BATCH_COL_BLOCKS ? (size_t)ti.z * g.N : 0);
  const int r_first = ti.m0 + row0 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = ti.n_tile * BN + 8 * j + 2 * (lane & 3);   // even, and n_total % 4 == 0: c + 1 is in range with c
    if (c >= p.n_total) continue;
    float2 bias2 = make_float2(0.f, 0.f);
    if (g.bias != nullptr) bias2 = __ldg(reinterpret_cast<const float2*>(g.bias + c));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r_first + 8 * i;
      if (r >= ti.row_end) continue;
      float x0 = acc[4 * j + 2 * i] + bias2.x, x1 = acc[4 * j + 2 * i + 1] + bias2.y;
      if (EPI == EPI_STORE) {
        *reinterpret_cast<float2*>(C + (size_t)r * g.ldc + c) = make_float2(apply_act(x0, g.act), apply_act(x1, g.act));
      } else if (EPI == EPI_GRU_ZR) {
        x0 = hard_sigmoid(x0); x1 = hard_sigmoid(x1);
        if (c < dgru) {
          *reinterpret_cast<float2*>(C + (size_t)r * g.ldc + c) = make_float2(x0, x1);   // z gate
        } else {
          const int cc = c - dgru;
          const float2 h = __ldg(reinterpret_cast<const float2*>(g.aux_h + (size_t)r * g.ld_h + cc));
          *reinterpret_cast<float2*>(g.C2 + (size_t)r * g.ldc2 + cc) = make_float2(x0 * h.x, x1 * h.y);
        }
      } else {  // EPI_GRU_OUT: h' = z*h + (1-z)*act(.)
        x0 = apply_act(x0, g.act); x1 = apply_act(x1, g.act);
        const float2 h = __ldg(reinterpret_cast<const float2*>(g.aux_h + (size_t)r * g.ld_h + c));
        const float2 zz = __ldg(reinterpret_cast<const float2*>(g.aux_z + (size_t)r * g.ld_z + c));
        *reinterpret_cast<float2*>(C + (size_t)r * g.ldc + c) =
            make_float2(zz.x * h.x + (1.0f - zz.x) * x0, zz.y * h.y + (1.0f - zz.y) * x1);
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------
// Persistent, warp-specialised kernel.  Roles (4 warpgroups):
//   warpgroups 0-1  consumers: wgmma on 64 rows each, epilogue from registers
//   warpgroups 2-3  A producers taking K chunks in turn; thread 0 of the producing group also issues the chunk's
//                   weight-image bulk copy
// Each CTA walks tiles  t = blockIdx.x, blockIdx.x + gridDim.x, ...  over one ring of S stages, so the producers
// load the next tile while the consumers write the current one back.
// GATHER: A rows follow an index list (GemmParams::a_rows: the compact (source, type) transform).
// -------------------------------------------------------------------------------------------------
template <int EPI, int BN, bool GATHER = false>
__global__ void __launch_bounds__(TC_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const GemmParams& g = p.g;
  const int tid = threadIdx.x, wg = tid >> 7;
  const int S = p.stages;
  constexpr int B_IMG_BYTES = BN * 128;
  constexpr int STAGE_BYTES = 2 * A_IMG_BYTES + 2 * B_IMG_BYTES;
  const int nchunks = p.chunks1 + p.chunks2;
  // shared-memory map (32-bit shared addresses): operand ring | full barriers | empty barriers
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = ring + (uint32_t)p.ring_bytes, empty0 = full0 + 8 * S;
  const int my_tiles = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, TC_GROUP_THREADS + 1);   // one producer group + the weight copy's expect_tx arrival
      mbar_init(empty0 + 8 * s, TC_CONSUMERS);          // one elected thread per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Everything above touched only this CTA's own state and may have run while the previous kernel of the stream was still
  // finishing (programmatic dependent launch); A, the weight images and C must not be touched before that kernel has completed.
  pdl_wait();
  pdl_launch_dependents();

  if (wg >= TC_CONSUMERS) {
    // =========================== A producers (+ weight-image copies) ===========================
    // Group g owns the chunks q = g, g+2, ... of this CTA's flat (tile, chunk) sequence.  A thread issues the loads of its
    // NEXT chunk right after publishing the current one, so they are in flight during the other group's time slot.
    const int group = wg - TC_CONSUMERS;
    const int ptid = tid & 127;
    // Groups in use: never more than ring stages.  A group that has published chunk q waits for the stage of chunk q + G; with
    // G > S that stage's "empty" barrier can still be TWO phases behind the awaited one, and an mbarrier parity wait cannot
    // tell "two behind" from "done" (the producer would overwrite a stage the tensor core has not read yet).
    const int ngroups = S < TC_GROUPS ? S : TC_GROUPS;
    const int total_q = group < ngroups ? my_tiles * nchunks : 0;
    auto load_a_chunk = [&](int q, float4 (&v)[8]) {
      const int ti_idx = q / nchunks, c = q - ti_idx * nchunks;
      const TileInfo ti = decode_tile(p, (int)blockIdx.x + ti_idx * (int)gridDim.x);
      const bool seg2 = c >= p.chunks1;
      const int k0 = (seg2 ? c - p.chunks1 : c) * TC_BK;
      const int Kseg = seg2 ? g.K2 : g.K1;
      const float* Abase = seg2 ? g.A2 : (g.batch_mode == BATCH_COL_BLOCKS ? g.A1 + (size_t)ti.z * g.K1 : g.A1);
      const int lda = seg2 ? g.lda2 : g.lda1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int f = ptid + i * TC_GROUP_THREADS;
        const int row = f >> 3, c16 = f & 7;
        const int grow = ti.m0 + row, gk = k0 + c16 * 4;
        if (GATHER) {
          const bool in = grow < ti.row_end && gk < Kseg;
          const int arow = in ? __ldg(g.a_rows + grow) : 0;
          v[i] = in ? __ldg(reinterpret_cast<const float4*>(Abase + (size_t)arow * lda + gk)) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
          v[i] = (grow < ti.row_end && gk < Kseg) ? __ldg(reinterpret_cast<const float4*>(Abase + (size_t)grow * lda + gk))
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    };
    float4 va[8];
    if (group < total_q) load_a_chunk(group, va);
    for (int q = group; q < total_q; q += ngroups) {
      const int s = q % S;
      const int use = q / S;
      if (use > 0) mbar_wait(empty0 + 8 * s, (use - 1) & 1);
      const uint32_t a_hi = ring + (uint32_t)(s * STAGE_BYTES);
      const uint32_t a_lo = a_hi + A_IMG_BYTES;
      if (ptid == 0) {   // the chunk's hi and lo weight images are adjacent in the packed buffer and in the stage
        const int ti_idx = q / nchunks, c = q - ti_idx * nchunks;
        const TileInfo ti = decode_tile(p, (int)blockIdx.x + ti_idx * (int)gridDim.x);
        const float* src = p.packed + (size_t)ti.z * p.packed_stride + ((size_t)ti.n_tile * nchunks + c) * 2 * (BN * TC_BK);
        mbar_arrive_expect_tx(full0 + 8 * s, 2 * B_IMG_BYTES);
        bulk_copy_g2s(a_hi + 2 * A_IMG_BYTES, src, 2 * B_IMG_BYTES, full0 + 8 * s);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int f = ptid + i * TC_GROUP_THREADS;
        const int row = f >> 3, c16 = f & 7;
        float4 hi, lo;
        split_tf32(va[i].x, hi.x, lo.x); split_tf32(va[i].y, hi.y, lo.y);
        split_tf32(va[i].z, hi.z, lo.z); split_tf32(va[i].w, hi.w, lo.w);
        const uint32_t off = (uint32_t)(row * 128 + ((c16 ^ (row & 7)) << 4));
        sts128(a_hi + off, hi);
        sts128(a_lo + off, lo);
      }
      fence_proxy_async_smem();                     // generic-proxy writes -> visible to the tensor core (async proxy)
      mbar_arrive(full0 + 8 * s);
      if (q + ngroups < total_q) load_a_chunk(q + ngroups, va);
    }
  } else {
    // =========================== consumers: wgmma + epilogue ===========================
    const int lane = tid & 31, warp_in_wg = (tid >> 5) & 3;
    const bool elected = (tid & 127) == 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    int q = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const TileInfo ti = decode_tile(p, (int)blockIdx.x + it * (int)gridDim.x);
      for (int c = 0; c < nchunks; ++c, ++q) {
        const int s = q % S;
        mbar_wait(full0 + 8 * s, (q / S) & 1);
        const uint32_t a_hi = ring + (uint32_t)(s * STAGE_BYTES) + (uint32_t)(wg * A_HALF_BYTES);
        const uint32_t a_lo = a_hi + A_IMG_BYTES;
        const uint32_t b_hi = ring + (uint32_t)(s * STAGE_BYTES + 2 * A_IMG_BYTES);
        const uint32_t b_lo = b_hi + B_IMG_BYTES;
        const uint64_t da_hi = make_sw128_desc(a_hi), da_lo = make_sw128_desc(a_lo);
        const uint64_t db_hi = make_sw128_desc(b_hi), db_lo = make_sw128_desc(b_lo);
        fence_operands(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 8; ++k) {       // k8 = 32 bytes: advance the start address by 2 (>>4 units)
          const uint64_t adv = (uint64_t)(k * 2);
          wgmma_tf32<BN>(acc, da_lo + adv, db_hi + adv, (c | k) != 0);   // small terms first
          wgmma_tf32<BN>(acc, da_hi + adv, db_lo + adv, 1);
          wgmma_tf32<BN>(acc, da_hi + adv, db_hi + adv, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();                            // the group of chunk q - 1 has retired: its stage is reusable
        fence_operands(acc);
        if (c > 0 && elected) mbar_arrive(empty0 + 8 * ((q - 1) % S));
      }
      wgmma_wait<0>();
      fence_operands(acc);
      if (elected) mbar_arrive(empty0 + 8 * ((q - 1) % S));
      epilogue_regs<EPI, BN>(p, ti, acc, wg * 64 + warp_in_wg * 16, lane);
    }
  }
}

int pick_bn(long m_tiles, int n_total, int gz) {
  int best = 32;
  double best_cost = 1e30;
  for (int bn = 128; bn >= 32; bn /= 2) {
    const long ctas = m_tiles * ((n_total + bn - 1) / bn) * gz;
    const long waves = (ctas + RGNN_WAVE_SMS - 1) / RGNN_WAVE_SMS;
    const double cost = (double)waves * (96.0 + bn);   // per-tile time ~ fixed overhead + columns
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

}  // namespace

// ---- optional cache of packed weight images (static weights: inference / benchmarking) ----------------
// Off by default.  Keyed by every input of the packing (weight pointers, leading dims, K/N, batching, BN);
// the caller promises not to modify cached weights in place without calling rgnn_weight_cache_clear().
struct PackKey {
  uint64_t h[4];
  bool operator==(const PackKey& o) const { return h[0] == o.h[0] && h[1] == o.h[1] && h[2] == o.h[2] && h[3] == o.h[3]; }
};
struct PackEntry { PackKey key; float* images; size_t bytes; };
static std::vector<PackEntry> g_pack_cache;
static std::mutex g_pack_mutex;
static bool g_pack_cache_on = false;

static inline void mix(uint64_t& h, uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); }
static PackKey make_pack_key(const GemmParams& g, int BN, int device) {
  PackKey k = {{0x1234, 0x5678, 0x9abc, (uint64_t)device}};
  const int nb = (g.batch_mode == BATCH_NONE) ? 1 : g.batch;
  for (int j = 0; j < nb; ++j) {
    const uint64_t a = (uint64_t)(g.batch_mode == BATCH_NONE ? g.B1 : g.bptr[j]);
    const uint64_t b = (uint64_t)(g.batch_mode == BATCH_NONE ? g.B2 : g.bptr2[j]);
    mix(k.h[j & 1], a); mix(k.h[2], b); mix(k.h[3], a * 31 + b + j);
  }
  mix(k.h[0], ((uint64_t)g.K1 << 32) | (uint32_t)g.K2);
  mix(k.h[1], ((uint64_t)g.N << 32) | (uint32_t)BN);
  mix(k.h[2], ((uint64_t)g.ldb1 << 32) | (uint32_t)g.ldb2);
  mix(k.h[3], ((uint64_t)g.batch_mode << 32) | (uint32_t)g.batch);
  return k;
}

void gemm_weight_cache_enable(bool on) { std::lock_guard<std::mutex> l(g_pack_mutex); g_pack_cache_on = on; }
void gemm_weight_cache_clear() {
  std::lock_guard<std::mutex> l(g_pack_mutex);
  for (auto& e : g_pack_cache) cudaFree(e.images);
  g_pack_cache.clear();
}
bool gemm_weight_cache_enabled() { return g_pack_cache_on; }

size_t gemm_tc_pack_bytes(const GemmParams& g) {
  if (g_pack_cache_on) return 1024;   // images live in the cache, the caller's scratch is not used
  return gemm_tc_pack_bytes_uncached(g);
}
size_t gemm_tc_pack_bytes_uncached(const GemmParams& g) {
  const int chunks = (g.K1 + TC_BK - 1) / TC_BK + (g.K2 + TC_BK - 1) / TC_BK;
  const int n_total = (g.batch_mode == BATCH_SHARED_A) ? g.batch * g.N : g.N;
  const int gz = (g.batch_mode == BATCH_ROW_RANGES || g.batch_mode == BATCH_COL_BLOCKS) ? g.batch : 1;
  const int rows = (g.batch_mode == BATCH_ROW_RANGES) ? g.max_rows : g.M;
  const int bn = pick_bn((rows + TC_BM - 1) / TC_BM, n_total, gz);
  const size_t tiles = (n_total + bn - 1) / bn;
  return align_up(tiles * chunks * 2 * (size_t)bn * TC_BK * sizeof(float) * gz, 1024);
}

int launch_gemm_tc(const GemmParams& g, void* pack_ws, size_t pack_ws_bytes, cudaStream_t stream) {
  RGNN_REQUIRE(g.M >= 0 && g.N > 0 && g.K1 > 0 && g.K2 >= 0, "gemm: bad dims M=%d N=%d K1=%d K2=%d", g.M, g.N, g.K1, g.K2);
  RGNN_REQUIRE((g.N % 4) == 0 && (g.K1 % 4) == 0 && (g.K2 % 4) == 0, "gemm: N, K must be multiples of 4 (N=%d K1=%d K2=%d)", g.N, g.K1, g.K2);
  RGNN_REQUIRE((g.lda1 % 4) == 0 && (g.ldb1 % 4) == 0 && (g.ldc % 4) == 0, "gemm: leading dims must keep 16-byte rows");
  RGNN_REQUIRE(g.batch >= 1 && g.batch <= RGNN_MAX_EDGE_TYPES, "gemm: batch %d out of range", g.batch);
  RGNN_REQUIRE(aligned16(g.A1) && aligned16(g.C) && (g.K2 == 0 || aligned16(g.A2)), "gemm: operands must be 16-byte aligned");
  RGNN_REQUIRE(g.bias == nullptr || aligned16(g.bias), "gemm: bias must be 16-byte aligned");
  const int rows = (g.batch_mode == BATCH_ROW_RANGES) ? g.max_rows : g.M;
  if (rows <= 0) return RGNN_OK;
  RGNN_REQUIRE(g.batch_mode != BATCH_K_BLOCKS_T || (g.k_block > 0 && g.K1 == g.batch * g.k_block && g.K2 == 0),
               "gemm: BATCH_K_BLOCKS_T needs K1 == batch * k_block and no second segment");
  if (g.a_rows != nullptr)
    RGNN_REQUIRE(g.epi == EPI_STORE && g.K2 == 0, "gemm: gathered A rows support the plain store epilogue and one K segment");

  TcParams p;
  p.g = g;
  p.chunks1 = (g.K1 + TC_BK - 1) / TC_BK;
  p.chunks2 = (g.K2 + TC_BK - 1) / TC_BK;
  const int nchunks = p.chunks1 + p.chunks2;
  p.n_total = (g.batch_mode == BATCH_SHARED_A) ? g.batch * g.N : g.N;
  const int gz = (g.batch_mode == BATCH_ROW_RANGES || g.batch_mode == BATCH_COL_BLOCKS) ? g.batch : 1;
  p.BN = pick_bn((rows + TC_BM - 1) / TC_BM, p.n_total, gz);
  const int n_tiles = (p.n_total + p.BN - 1) / p.BN;
  p.n_tiles = n_tiles;
  auto tiles_of = [&](int nrows) { return ((nrows + TC_BM - 1) / TC_BM) * n_tiles; };
  // tile table: batch entry z owns tiles [tile_start[z], tile_start[z+1])
  p.tile_start[0] = 0;
  if (g.batch_mode == BATCH_ROW_RANGES) {
    for (int z = 0; z < g.batch; ++z) p.tile_start[z + 1] = p.tile_start[z] + tiles_of(g.row_off[z + 1] - g.row_off[z]);
    p.total_tiles = p.tile_start[g.batch];
  } else if (g.batch_mode == BATCH_COL_BLOCKS) {
    for (int z = 0; z < g.batch; ++z) p.tile_start[z + 1] = p.tile_start[z] + tiles_of(g.M);
    p.total_tiles = p.tile_start[g.batch];
  } else {
    p.total_tiles = tiles_of(g.M);
    p.tile_start[1] = p.total_tiles;
  }
  if (p.total_tiles <= 0) return RGNN_OK;

  const size_t stage_bytes = 2 * (size_t)A_IMG_BYTES + 2 * (size_t)p.BN * 128;
  p.stages = (int)(TC_RING_BUDGET / stage_bytes);
  if (p.stages > 4) p.stages = 4;
  if (p.stages < 1) p.stages = 1;
  p.ring_bytes = (int)(p.stages * stage_bytes);
  p.packed_stride = (size_t)n_tiles * nchunks * 2 * p.BN * TC_BK;
  const size_t need = align_up(p.packed_stride * sizeof(float) * gz, 1024);
  bool need_pack = true;
  if (g_pack_cache_on) {
    int device = 0;
    cudaGetDevice(&device);
    const PackKey key = make_pack_key(g, p.BN, device);
    std::lock_guard<std::mutex> l(g_pack_mutex);
    float* images = nullptr;
    for (auto& e : g_pack_cache)
      if (e.key == key && e.bytes == need) { images = e.images; need_pack = false; break; }
    if (images == nullptr) {
      cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
      cudaStreamIsCapturing(stream, &cap);
      RGNN_REQUIRE(cap == cudaStreamCaptureStatusNone, "gemm: weight cache miss during CUDA-graph capture (run the layer once eagerly first)");
      RGNN_CHECK_CUDA(cudaMalloc(&images, need));
      g_pack_cache.push_back({key, images, need});
    }
    pack_ws = images;
  } else {
    RGNN_REQUIRE(pack_ws != nullptr && pack_ws_bytes >= need && (reinterpret_cast<uintptr_t>(pack_ws) & 15u) == 0,
                 "gemm: weight-image workspace too small (%zu < %zu)", pack_ws_bytes, need);
  }
  p.packed = static_cast<const float*>(pack_ws);

  // ---- pack the weights into shared-memory images ----
  for (int zz = 0; need_pack && zz < gz; ++zz) {
    PackParams q;
    q.ldb1 = g.ldb1; q.ldb2 = g.ldb2; q.K1 = g.K1; q.K2 = g.K2;
    q.BN = p.BN; q.chunks1 = p.chunks1; q.chunks2 = p.chunks2;
    q.n_total = p.n_total;
    q.transposed = 0; q.k_block = 0;
    if (g.batch_mode == BATCH_K_BLOCKS_T) {
      q.transposed = 1; q.k_block = g.k_block; q.block_cols = g.N;
      for (int j = 0; j < g.batch; ++j) { q.b1[j] = g.bptr[j]; q.b2[j] = nullptr; }
    } else if (g.batch_mode == BATCH_SHARED_A) {
      q.block_cols = g.N;
      for (int j = 0; j < g.batch; ++j) { q.b1[j] = g.bptr[j]; q.b2[j] = g.bptr2[j]; }
    } else if (g.batch_mode == BATCH_NONE) {
      q.block_cols = g.N; q.b1[0] = g.B1; q.b2[0] = g.B2;
    } else {
      q.block_cols = g.N; q.b1[0] = g.bptr[zz]; q.b2[0] = g.bptr2[zz];
    }
    for (int j = 0; j < ((g.batch_mode == BATCH_SHARED_A || g.batch_mode == BATCH_K_BLOCKS_T) ? g.batch : 1); ++j) {
      RGNN_REQUIRE(q.b1[j] != nullptr && (g.K2 == 0 || q.b2[j] != nullptr), "gemm: weight pointer %d is NULL", j);
    }
    q.out = static_cast<float*>(pack_ws) + (size_t)zz * p.packed_stride;
    RGNN_CHECK_CUDA(launch_pdl(pack_b_kernel, dim3(nchunks, n_tiles, (p.BN + 31) / 32), dim3(256), 0, stream, q));
    RGNN_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }

  const size_t smem = 1024 + (size_t)p.ring_bytes + 2 * p.stages * sizeof(uint64_t);
  // per-DEVICE launch state (a process may drive several GPUs): SM count, opt-in shared memory
  constexpr int MAX_DEV = 64;
  static int num_sms_of[MAX_DEV] = {};
  int device = 0;
  cudaGetDevice(&device);
  const int dv = (device >= 0 && device < MAX_DEV) ? device : 0;
  if (num_sms_of[dv] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    num_sms_of[dv] = n > 0 ? n : RGNN_WAVE_SMS;
  }
  const int num_sms = num_sms_of[dv];

  using KernelFn = void (*)(TcParams);
  // [gather + epilogue][BN]: slots 0-2 the epilogues, slot 3 the gathered-rows store
  static const KernelFn table[4][3] = {
      {gemm_wgmma_kernel<EPI_STORE, 32>, gemm_wgmma_kernel<EPI_STORE, 64>, gemm_wgmma_kernel<EPI_STORE, 128>},
      {gemm_wgmma_kernel<EPI_GRU_ZR, 32>, gemm_wgmma_kernel<EPI_GRU_ZR, 64>, gemm_wgmma_kernel<EPI_GRU_ZR, 128>},
      {gemm_wgmma_kernel<EPI_GRU_OUT, 32>, gemm_wgmma_kernel<EPI_GRU_OUT, 64>, gemm_wgmma_kernel<EPI_GRU_OUT, 128>},
      {gemm_wgmma_kernel<EPI_STORE, 32, true>, gemm_wgmma_kernel<EPI_STORE, 64, true>, gemm_wgmma_kernel<EPI_STORE, 128, true>}};
  const int slot = g.a_rows != nullptr ? 3 : g.epi;
  const int bn_idx = p.BN == 32 ? 0 : p.BN == 64 ? 1 : 2;
  KernelFn fn = table[slot][bn_idx];
  static bool attr_done[MAX_DEV][4][3] = {};
  if (!attr_done[dv][slot][bn_idx]) {
    RGNN_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM_MAX));
    attr_done[dv][slot][bn_idx] = true;
  }
  const int ctas = p.total_tiles < num_sms ? p.total_tiles : num_sms;   // persistent: at most one CTA per SM
  RGNN_CHECK_CUDA(launch_pdl(fn, dim3((unsigned)ctas), dim3(TC_THREADS), smem, stream, p));
  RGNN_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return RGNN_OK;
}

}  // namespace rgnn
