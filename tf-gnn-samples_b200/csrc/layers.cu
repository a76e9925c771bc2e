// layers.cu -- C-ABI entry points: one forward per reference layer function (include/rgnn.h).
//
// Every layer is re-associated "transform first" (SURVEY.md 7): the per-type Dense is applied to the
// V node rows (one tensor-core GEMM over all types, T = H . [W_0|...|W_{L-1}]) instead of to the M
// gathered edge rows (gnns/rgcn.py:88,98 does M*D*D*2 FLOP; this does V*L*D*D*2), and the edge stage
// is one fused sorted-segment kernel (seg_kernels.cu).  RGAT already works this way in the reference
// (rgat.py:95-96).  Only an MLP's layers after a per-edge nonlinearity stay per-edge (edge-MLP with
// >= 1 hidden layer and target input): those run as per-type row-range GEMMs over materialised rows.
#include <algorithm>
#include <mutex>
#include <atomic>
#include <utility>
#include <vector>
#include <string.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm.cuh"
#include "plan.cuh"
#include "seg.cuh"

namespace rgnn {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

namespace {

// bump allocator over the caller's workspace
struct Arena {
  char* base;
  size_t cap, used = 0;
  bool overflow = false;
  Arena(void* b, size_t c) : base(static_cast<char*>(b)), cap(c) {}
  float* floats(size_t n) {
    const size_t bytes = align_up(n * sizeof(float), 256);
    if (base == nullptr || used + bytes > cap) { overflow = true; used += bytes; return nullptr; }
    float* p = reinterpret_cast<float*>(base + used);
    used += bytes;
    return p;
  }
};

int check_common(const rgnn_plan_t* plan, const float* h, int d_in, int d_out, const float* out, int num_timesteps,
                 const char* who) {
  RGNN_REQUIRE(plan != nullptr, "%s: plan is NULL", who);
  RGNN_REQUIRE(h != nullptr && out != nullptr, "%s: node_embeddings / out is NULL", who);
  RGNN_REQUIRE(h != out, "%s: out must not alias node_embeddings", who);
  RGNN_REQUIRE(aligned16(h) && aligned16(out), "%s: node_embeddings / out must be 16-byte aligned", who);
  RGNN_REQUIRE(d_in > 0 && d_out > 0 && (d_in % 4) == 0 && (d_out % 4) == 0,
               "%s: state dims must be positive multiples of 4 (d_in=%d, d_out=%d)", who, d_in, d_out);
  RGNN_REQUIRE(num_timesteps >= 1, "%s: num_timesteps %d < 1", who, num_timesteps);
  RGNN_REQUIRE(num_timesteps == 1 || plan->Vt == plan->V,
               "%s: a plan restricted to %d of %d target rows supports num_timesteps == 1 only (halo rows are not updated)", who, plan->Vt, plan->V);
  RGNN_REQUIRE(num_timesteps == 1 || d_in == d_out,
               "%s: num_timesteps > 1 needs state_dim == input dim (d_in=%d, d_out=%d)", who, d_in, d_out);
  return RGNN_OK;
}
int check_act(int act, const char* who) {
  RGNN_REQUIRE(act >= RGNN_ACT_LINEAR && act <= RGNN_ACT_GELU, "%s: Unknown activation function code %d", who, act);
  return RGNN_OK;
}
int check_agg(int agg, const char* who) {
  RGNN_REQUIRE(agg >= RGNN_AGG_SUM && agg <= RGNN_AGG_SQRT_N, "%s: Unknown aggregation function code %d", who, agg);
  return RGNN_OK;
}
// rgnn_workspace_bytes sizes every scratch row of an MLP layer by max(2 d_in, d_out): a wider MLP layer is refused up
// front, before anything is enqueued, instead of failing for lack of workspace halfway through the call.
int check_mlp_widths(const int32_t* dims, int nl, int d_in, int d_out, const char* what, const char* who) {
  const int limit = (2 * d_in > d_out) ? 2 * d_in : d_out;
  for (int j = 1; j <= nl; ++j) {
    if (dims[j] > limit) {
      set_error("%s: %s layer %d has width %d, above this build's limit max(2 * d_in, d_out) = %d", who, what, j - 1, dims[j], limit);
      return RGNN_E_UNSUPPORTED;
    }
  }
  return RGNN_OK;
}
int check_ws(const Arena& a, const char* who) {
  if (a.overflow) {
    set_error("%s: workspace too small (%zu bytes given, %zu needed)", who, a.cap, a.used);
    return RGNN_E_WORKSPACE;
  }
  return RGNN_OK;
}

// Dispatch one dense contraction on the wgmma kernel (weight images packed into arena scratch that is released
// right after the enqueue -- later users are stream-ordered).
int run_gemm(const GemmParams& g, Arena& ar, cudaStream_t stream) {
  const size_t need = gemm_tc_pack_bytes(g);
  const size_t mark = ar.used;
  void* ws = ar.floats(need / sizeof(float));
  if (ar.overflow) {
    set_error("workspace too small for the weight images of a dense contraction (%zu bytes given, %zu needed)", ar.cap, ar.used);
    return RGNN_E_WORKSPACE;
  }
  const int rc = launch_gemm_tc(g, ws, need, stream);
  ar.used = mark;
  return rc;
}

// T[V, batch*N] = A[V, K] . B_z  for z < batch  (shared A)
int gemm_shared_a(Arena& ar, const float* A, int V, int K, const float* const* B, int batch, int ldb, int N, float* C, int act,
                  cudaStream_t stream) {
  GemmParams g;
  g.A1 = A; g.lda1 = K; g.K1 = K;
  g.M = V; g.N = N;
  g.C = C; g.ldc = batch * N;
  g.ldb1 = ldb;
  g.act = act;
  g.batch_mode = BATCH_SHARED_A; g.batch = batch;
  for (int z = 0; z < batch; ++z) { g.bptr[z] = B[z]; g.bptr2[z] = nullptr; }
  return run_gemm(g, ar, stream);
}

// The per-type Dense on the SOURCE side of the edge stage (rgcn.py:98, ggnn.py:80-82, gnn_film.py:94 applied to nodes).
// Dense form: T[V, L, D] = cur . [W_0|..|W_{L-1}].  Sparsely typed graphs (the plan holds a compact pair table, plan.cuh):
// only the (source, type) rows that some edge gathers are transformed -- a row-range GEMM per type whose A rows follow the
// pair list -- and the edge stage addresses the compact table.  Call after seg_from_plan(s, plan).
int transform_sources(const rgnn_plan_t* plan, Arena& ar, const float* cur, int d_in, int D, const float* const* W, float* T,
                      cudaStream_t stream, SegParams& s) {
  const int V = plan->V, L = plan->L;
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));   // an overlapped halo exchange must have landed before source rows are read
  if (plan->n_pairs >= 0 && plan->pair_src != nullptr) {
    GemmParams g;
    g.A1 = cur; g.lda1 = d_in; g.K1 = d_in; g.a_rows = plan->pair_src;
    g.M = plan->n_pairs; g.N = D; g.C = T; g.ldc = D; g.ldb1 = D;
    g.batch_mode = BATCH_ROW_RANGES; g.batch = L; g.max_rows = plan->max_type_pairs;
    for (int l = 0; l < L; ++l) { g.bptr[l] = W[l]; g.bptr2[l] = nullptr; g.row_off[l] = plan->pair_type_off[l]; }
    g.row_off[L] = plan->pair_type_off[L];
    RGNN_PROPAGATE(run_gemm(g, ar, stream));
    s.table = T; s.e_idx = plan->e_pair; s.stride_idx = D; s.stride_type = 0;
    return RGNN_OK;
  }
  RGNN_PROPAGATE(gemm_shared_a(ar, cur, V, d_in, W, L, D, D, T, RGNN_ACT_LINEAR, stream));
  s.table = T; s.stride_idx = (long)L * D; s.stride_type = D;
  return RGNN_OK;
}
// the weight-image scratch transform_sources() takes from the arena (sized before anything is enqueued)
size_t transform_sources_pack_bytes(const rgnn_plan_t* plan, int d_in, int D) {
  GemmParams g;
  g.K1 = d_in; g.N = D; g.batch = plan->L;
  if (plan->n_pairs >= 0 && plan->pair_src != nullptr) {
    g.batch_mode = BATCH_ROW_RANGES; g.M = plan->n_pairs; g.max_rows = plan->max_type_pairs;
  } else {
    g.batch_mode = BATCH_SHARED_A; g.M = plan->V;
  }
  return gemm_tc_pack_bytes(g);
}

// scratch for the multi-CTA split of heavy targets (seg_kernels.cu); nothing when the plan is known to have none
size_t heavy_scratch_floats(const rgnn_plan_t* plan, size_t d) {
  return plan->num_heavy_host == 0 ? 0 : (size_t)plan->heavy_items_cap * d;
}
void seg_heavy_scratch(SegParams& s, const rgnn_plan_t* plan, Arena& ar, int d) {
  if (plan->num_heavy_host == 0 || plan->heavy_items == nullptr) return;
  float* scratch = ar.floats((size_t)plan->heavy_items_cap * d);
  if (ar.overflow) return;   // the caller's check_ws reports it
  s.heavy_scratch = scratch;
}

void seg_from_plan(SegParams& s, const rgnn_plan_t* plan) {
  s.V = plan->Vt; s.L = plan->L; s.scale_ld = plan->V;   // only the wanted target rows are reduced (rgnn_plan_set_num_targets)
  s.heavy_list = plan->heavy_list; s.heavy_count = plan->err_flag + 1;
  s.heavy_base = plan->heavy_base; s.heavy_items = plan->heavy_items; s.heavy_item_count = plan->err_flag + 3;
  s.heavy_items_known = plan->num_heavy_items_host; s.heavy_items_cap = plan->heavy_items_cap; s.heavy_chunk = RGNN_HEAVY_CHUNK;
  s.heavy_threshold = RGNN_HEAVY_SEGMENT; s.heavy_known = plan->num_heavy_host;
  s.seg_off = plan->seg_off; s.e_type = plan->e_type; s.e_idx = plan->e_src;
}

// Where the per-message rows of an MLP-style layer live after the dense stages.
struct MsgSource {
  const float* table = nullptr;
  const int32_t* idx = nullptr;
  long stride_idx = 0, stride_type = 0;
  int width = 0;
  int msg_mode = MSG_LINEAR;
  const float* mod_table = nullptr;
  long mod_sn = 0, mod_st = 0;
};

// Evaluate MLP_l([h_u | h_v]) / MLP_l(h_u) for every message (gnn_edge_mlp.py:87-102, rgin.py:106-124).
// kernels: type-major [L][nl]; dims [nl+1]; nl = number of Dense kernels (hidden layers + 1), 0 = no MLP.
int build_mlp_messages(const rgnn_plan_t* plan, const float* cur, int d_in, const float* const* kernels,
                       const int32_t* dims, int nl, int use_target, int hidden_act, Arena& ar, cudaStream_t stream,
                       MsgSource* out) {
  const int V = plan->V, L = plan->L;
  const int M = (int)plan->M;
  MsgSource ms;
  if (nl == 0) {
    if (!use_target) {
      ms.table = cur; ms.idx = plan->e_src; ms.stride_idx = d_in; ms.stride_type = 0; ms.width = d_in;
    } else {   // messages are the raw [h_u | h_v] pairs (rgin.py:114-124 with edge MLP None)
      float* X = ar.floats((size_t)M * 2 * d_in);
      if (ar.overflow) { *out = ms; return RGNN_OK; }
      EdgeBuildParams b;
      b.L = L; b.D = d_in; b.o_src = plan->o_src; b.o_tgt = plan->o_tgt;
      memcpy(b.type_off, plan->type_off, sizeof(b.type_off)); b.max_type_edges = plan->max_type_edges;
      b.p = cur; b.p_stride_node = d_in; b.p_stride_type = 0; b.concat = 1;
      b.x = X; b.ldx = 2 * d_in;
      RGNN_PROPAGATE(launch_edge_build(b, stream));
      ms.table = X; ms.idx = plan->e_orig; ms.stride_idx = 2 * d_in; ms.stride_type = 0; ms.width = 2 * d_in;
    }
    *out = ms;
    return RGNN_OK;
  }
  RGNN_REQUIRE(nl <= RGNN_MAX_MLP_LAYERS, "edge MLP with %d layers exceeds the supported %d", nl, RGNN_MAX_MLP_LAYERS);
  RGNN_REQUIRE(dims[0] == d_in * (use_target ? 2 : 1), "edge MLP input dim %d does not match %d", dims[0],
               d_in * (use_target ? 2 : 1));
  for (int j = 1; j <= nl; ++j) RGNN_REQUIRE(dims[j] > 0 && (dims[j] % 4) == 0, "edge MLP dim %d must be a positive multiple of 4", dims[j]);
  for (int i = 0; i < L * nl; ++i) RGNN_REQUIRE(kernels[i] != nullptr, "edge MLP kernel %d is NULL", i);

  const float* bp[RGNN_MAX_EDGE_TYPES];
  if (!use_target) {
    // whole MLP is per (node, type): chain of node-level GEMMs
    float* prev = ar.floats((size_t)V * L * dims[1]);
    if (ar.overflow) { *out = ms; return RGNN_OK; }
    for (int l = 0; l < L; ++l) bp[l] = kernels[l * nl + 0];
    RGNN_PROPAGATE(gemm_shared_a(ar, cur, V, d_in, bp, L, dims[1], dims[1], prev, nl > 1 ? hidden_act : RGNN_ACT_LINEAR, stream));
    for (int j = 1; j < nl; ++j) {
      float* next = ar.floats((size_t)V * L * dims[j + 1]);
      if (ar.overflow) { *out = ms; return RGNN_OK; }
      GemmParams g;
      g.A1 = prev; g.lda1 = L * dims[j]; g.K1 = dims[j];
      g.M = V; g.N = dims[j + 1]; g.C = next; g.ldc = L * dims[j + 1]; g.ldb1 = dims[j + 1];
      g.act = (j < nl - 1) ? hidden_act : RGNN_ACT_LINEAR;
      g.batch_mode = BATCH_COL_BLOCKS; g.batch = L;
      for (int l = 0; l < L; ++l) { g.bptr[l] = kernels[l * nl + j]; g.bptr2[l] = nullptr; }
      RGNN_PROPAGATE(run_gemm(g, ar, stream));
      prev = next;
    }
    ms.table = prev; ms.idx = plan->e_src; ms.stride_idx = (long)L * dims[nl]; ms.stride_type = dims[nl]; ms.width = dims[nl];
    *out = ms;
    return RGNN_OK;
  }
  // use_target: first Dense splits into a source half P and a target half Q of the kernel rows
  RGNN_REQUIRE(2 * L <= RGNN_MAX_EDGE_TYPES, "edge MLP with target input supports at most %d edge types", RGNN_MAX_EDGE_TYPES / 2);
  const int d1 = dims[1];
  float* PQ = ar.floats((size_t)V * 2 * L * d1);
  if (ar.overflow) { *out = ms; return RGNN_OK; }
  for (int l = 0; l < L; ++l) {
    bp[l] = kernels[l * nl + 0];                              // rows [0, d_in)      multiply h_u
    bp[L + l] = kernels[l * nl + 0] + (size_t)d_in * d1;      // rows [d_in, 2 d_in) multiply h_v
  }
  RGNN_PROPAGATE(gemm_shared_a(ar, cur, V, d_in, bp, 2 * L, d1, d1, PQ, RGNN_ACT_LINEAR, stream));
  if (nl == 1) {
    ms.table = PQ; ms.idx = plan->e_src; ms.stride_idx = 2L * L * d1; ms.stride_type = d1; ms.width = d1;
    ms.msg_mode = MSG_ADDTGT; ms.mod_table = PQ + (size_t)L * d1; ms.mod_sn = 2L * L * d1; ms.mod_st = d1;
    *out = ms;
    return RGNN_OK;
  }
  float* X = ar.floats((size_t)M * d1);
  if (ar.overflow) { *out = ms; return RGNN_OK; }
  {
    EdgeBuildParams b;
    b.L = L; b.D = d1; b.o_src = plan->o_src; b.o_tgt = plan->o_tgt;
    memcpy(b.type_off, plan->type_off, sizeof(b.type_off)); b.max_type_edges = plan->max_type_edges;
    b.p = PQ; b.p_stride_node = 2L * L * d1; b.p_stride_type = d1;
    b.q = PQ + (size_t)L * d1; b.q_stride_node = 2L * L * d1; b.q_stride_type = d1;
    b.act = hidden_act; b.x = X; b.ldx = d1;
    RGNN_PROPAGATE(launch_edge_build(b, stream));
  }
  float* prev = X;
  for (int j = 1; j < nl; ++j) {
    float* next = ar.floats((size_t)M * dims[j + 1]);
    if (ar.overflow) { *out = ms; return RGNN_OK; }
    GemmParams g;
    g.A1 = prev; g.lda1 = dims[j]; g.K1 = dims[j];
    g.M = M; g.N = dims[j + 1]; g.C = next; g.ldc = dims[j + 1]; g.ldb1 = dims[j + 1];
    g.act = (j < nl - 1) ? hidden_act : RGNN_ACT_LINEAR;
    g.batch_mode = BATCH_ROW_RANGES; g.batch = L; g.max_rows = plan->max_type_edges;
    for (int l = 0; l < L; ++l) { g.bptr[l] = kernels[l * nl + j]; g.bptr2[l] = nullptr; g.row_off[l] = plan->type_off[l]; }
    g.row_off[L] = plan->type_off[L];
    RGNN_PROPAGATE(run_gemm(g, ar, stream));
    prev = next;
  }
  ms.table = prev; ms.idx = plan->e_orig; ms.stride_idx = dims[nl]; ms.stride_type = 0; ms.width = dims[nl];
  *out = ms;
  return RGNN_OK;
}

void seg_from_source(SegParams& s, const MsgSource& ms) {
  s.table = ms.table; s.e_idx = ms.idx; s.stride_idx = ms.stride_idx; s.stride_type = ms.stride_type;
  s.D = ms.width; s.msg_mode = ms.msg_mode; s.mod_table = ms.mod_table;
  s.mod_stride_node = ms.mod_sn; s.mod_stride_type = ms.mod_st;
}

}  // namespace
}  // namespace rgnn

using namespace rgnn;

extern "C" int rgnn_version(void) { return RGNN_VERSION; }
extern "C" const char* rgnn_last_error(void) { return g_err; }
extern "C" int64_t rgnn_launch_count(void) { return (int64_t)g_launches.load(); }

extern "C" int rgnn_set_weight_cache(int enable) {
  gemm_weight_cache_enable(enable != 0);
  if (!enable) gemm_weight_cache_clear();
  return RGNN_OK;
}
extern "C" int rgnn_weight_cache_clear(void) {
  gemm_weight_cache_clear();
  return RGNN_OK;
}

extern "C" size_t rgnn_workspace_bytes(const rgnn_plan_t* plan, int layer_kind, int32_t d_in, int32_t d_out,
                                       int32_t mlp_layers) {
  if (plan == nullptr || d_in <= 0 || d_out <= 0) return 0;
  const size_t V = (size_t)plan->V, L = (size_t)plan->L, M = (size_t)plan->M;
  const size_t dm = (size_t)((2 * d_in > d_out) ? 2 * d_in : d_out);
  const size_t pad = 256 * 32;
  size_t floats = 0;
  switch (layer_kind) {
    case RGNN_LAYER_RGCN: floats = V * 2 * L * dm + 2 * V * dm; break;
    case RGNN_LAYER_GGNN: floats = V * L * dm + 6 * V * dm; break;
    case RGNN_LAYER_RGAT: floats = V * L * dm + 2 * V * L * dm / 4 + 2 * V * dm; break;
    case RGNN_LAYER_FILM: floats = 3 * V * L * dm + 2 * V * dm; break;
    case RGNN_LAYER_RGCN_BACKWARD: floats = 2 * V * L * dm + 2 * V * dm + (RGNN_WAVE_SMS * 16384 + L * dm * dm) + 64 * 1024; break;   // + split-K partial tiles of dW
    case RGNN_LAYER_EDGE_MLP:
    case RGNN_LAYER_RGIN: {
      const size_t nl = (size_t)(mlp_layers > 0 ? mlp_layers : 1);
      floats = V * 2 * L * dm * (nl + 1) + M * dm * (nl + 1) + (4 + nl) * V * dm;
      break;
    }
    case RGNN_LAYER_RGDCN: floats = V * L * dm * (size_t)(mlp_layers > 0 ? mlp_layers : 16) + 2 * V * dm; break;   // mlp_layers carries channel_dim
    case RGNN_LAYER_FILM_BACKWARD: {   // T, dT [V, L, D]; FW, dFW [Vt <= V, L, 2D]; d_a [Vt, D]; the second d_h term [Vt, d_in];
      const size_t di = (size_t)d_in, dd = (size_t)d_out;   // LN partials; split-K tiles of d_W / d_F
      floats = 6 * V * L * dd + V * (dd + di) + (size_t)FILM_LN_MAX_BLOCKS * 2 * dd + (RGNN_WAVE_SMS * 16384 + 2 * L * di * dd) + 64 * 1024;
      break;
    }
    case RGNN_LAYER_RGAT_BACKWARD: {   // T, dT [V, L, D]; s_src, s_tgt, D_src, D_tgt [<= V, L, K]; d_o [Vt, D]; m, den, c [Vt, K]
      const size_t di = (size_t)d_in, dd = (size_t)d_out;   // (K <= D / 4); d_att partials; split-K tiles of d_W
      floats = 3 * V * L * dd + 2 * V * dd + (size_t)RGAT_ATT_MAX_BLOCKS * L * 2 * dd + (RGNN_WAVE_SMS * 16384 + L * di * dd) + 64 * 1024;
      break;
    }
    case RGNN_LAYER_GGNN_BACKWARD: {   // T, then dT [V, L, D]; m, dm [V, D]; a, da [Vt, 3D]; rh, d(rh) / f, e [Vt, D];
      const size_t dd = (size_t)d_out;   // bias partials; split-K tiles of d_W / d_K / d_R
      floats = V * L * dd + 11 * V * dd + (size_t)GGNN_COLSUM_MAX_BLOCKS * 3 * dd + (RGNN_WAVE_SMS * 16384 + (L + 3) * dd * dd) + 64 * 1024;
      break;
    }
    case RGNN_LAYER_RGIN_BACKWARD: {   // Z_j, A_j and dQ / dA [V, L, <= dm] (at most 2 nl of them); a / d_a [V, dm];
      const size_t nl = (size_t)(mlp_layers > 0 ? mlp_layers : 1), dd = (size_t)d_out;   // U_k, Y_k, n [Vt <= V, dm];
      floats = 2 * nl * V * L * dm + (2 * nl + 2) * V * dm + (size_t)FILM_LN_MAX_BLOCKS * 2 * dd   // LN partials;
               + (RGNN_WAVE_SMS * 16384 + L * dm * dm) + 64 * 1024;                             // split-K tiles of d_E / d_K
      break;
    }
    case RGNN_LAYER_RGDCN_BACKWARD: {   // mlp_layers carries channel_dim K; P / dP [Vt, L, d K]; dS, dQ [V, L, d];
      const size_t Vt = (size_t)plan->Vt, dd = (size_t)d_out, Kc = (size_t)(mlp_layers > 0 ? mlp_layers : 16), KK = Kc * Kc;
      const size_t C = dd / Kc > 0 ? dd / Kc : 1, Q = std::min(L * C, (size_t)RGNN_MAX_EDGE_TYPES) * KK;   // d_h term [Vt, d];
      floats = Vt * L * dd * Kc + 2 * V * L * dd + Vt * dd + Vt * L * KK   // dP summed over channels [Vt, L, K K];
               + (RGNN_WAVE_SMS * 16384 + dd * Q)                         // split-K tiles of dF;
               + 2 * (Q + 128) * (dd + 128) + 1024;                       // weight images of the largest GEMM
      const size_t fwd_pack = 2 * (2 * dm + 64) * (2 * L * dm + 2 * dm + 512);
      return (floats + fwd_pack) * sizeof(float) + pad;   // no heavy-target scratch: nothing sized by M
    }
    default: return 0;
  }
  // scratch for the pre-swizzled hi/lo weight images of the largest dense contraction of the layer
  const size_t pack = 2 * (2 * dm + 64) * (2 * L * dm + 2 * dm + 512);
  floats += heavy_scratch_floats(plan, dm) + 64;   // partial rows of split heavy targets
  return (floats + pack) * sizeof(float) + pad;
}

// ---------------------------------------------------------------------------------------------
// gnns/rgcn.py:8-117
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_rgcn_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                 const float* const* edge_weights, const float* num_incoming, int activation,
                                 int aggregation, int normalize, int both, int num_timesteps, float* out,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "rgcn"));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));
  RGNN_PROPAGATE(check_act(activation, "rgcn"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgcn"));
  RGNN_REQUIRE(edge_weights != nullptr, "rgcn: edge_weights is NULL");
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "rgcn: normalize_by_num_incoming needs type_to_num_incoming_edges");
  const int V = plan->V, L = plan->L;
  RGNN_REQUIRE(!both || 2 * L <= RGNN_MAX_EDGE_TYPES, "rgcn: use_both_source_and_target supports at most %d edge types", RGNN_MAX_EDGE_TYPES / 2);
  for (int l = 0; l < L; ++l) RGNN_REQUIRE(edge_weights[l] != nullptr, "rgcn: edge weight %d is NULL", l);
  Arena ar(workspace, workspace_bytes);
  const int nb = both ? 2 * L : L;
  float* T = ar.floats((size_t)V * nb * d_out);
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * d_out); buf[1] = ar.floats((size_t)V * d_out); }
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, d_out);
  RGNN_PROPAGATE(check_ws(ar, "rgcn"));

  const float* bp[RGNN_MAX_EDGE_TYPES];
  const float* cur = h;
  int din = d_in;
  for (int t = 0; t < num_timesteps; ++t) {                                   // rgcn.py:81
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    for (int l = 0; l < L; ++l) {
      bp[l] = edge_weights[l];                                                // kernel rows [0, d_in): source half
      if (both) bp[L + l] = edge_weights[l] + (size_t)din * d_out;            // rows [d_in, 2 d_in): target half (rgcn.py:95)
    }
    SegParams s;
    seg_from_plan(s, plan);
    s.D = d_out;
    if (both) {
      RGNN_PROPAGATE(gemm_shared_a(ar, cur, V, din, bp, nb, d_out, d_out, T, RGNN_ACT_LINEAR, stream));   // rgcn.py:98 on nodes
      s.table = T; s.stride_idx = (long)nb * d_out; s.stride_type = d_out;
    } else {
      RGNN_PROPAGATE(transform_sources(plan, ar, cur, din, d_out, bp, T, stream, s));                     // rgcn.py:98 on the used (source, type) rows
    }
    s.num_incoming = normalize ? num_incoming : nullptr;                      // rgcn.py:100-104
    if (both) { s.msg_mode = MSG_ADDTGT; s.mod_table = T + (size_t)L * d_out; s.mod_stride_node = (long)nb * d_out; s.mod_stride_type = d_out; }
    s.agg = aggregation; s.act_out = activation;                              // rgcn.py:110,114
    s.out = dst; s.ld_out = d_out; s.heavy_scratch = heavy.heavy_scratch;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    cur = dst; din = d_out;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_rgcn_layer (source-only messages): what tf.gradients produces for
// gnns/rgcn.py:84-114 (the reference trains through TF autodiff, models/sparse_graph_model.py:253-260).
//   d_agg = grad_out * act'(.) / div            (elementwise)
//   d_T[u, l, :] = sum_{(u->v) in A_l} s_{l,v} * d_agg[v, :]      (sorted-segment kernel over the reverse index)
//   d_H = d_T . [W_0|...|W_{L-1}]^T             (wgmma GEMM, transposed weight images)
//   d_W_l = H^T . d_T[:, l, :]                  (TN wgmma GEMM, split-K with a deterministic two-stage sum)
extern "C" int rgnn_rgcn_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d_in, int32_t d_out,
                                  const float* const* edge_weights, const float* num_incoming, int activation,
                                  int aggregation, int normalize, const float* out, const float* grad_out,
                                  float* grad_h, float* const* grad_edge_weights, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr && h != nullptr && out != nullptr && grad_out != nullptr && edge_weights != nullptr,
               "rgcn_backward: NULL argument");
  RGNN_REQUIRE(d_in > 0 && d_out > 0 && (d_in % 4) == 0 && (d_out % 4) == 0, "rgcn_backward: dims must be positive multiples of 4");
  RGNN_PROPAGATE(check_act(activation, "rgcn_backward"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgcn_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("rgcn_backward: the gradient of 'max' aggregation is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "rgcn_backward: normalize_by_num_incoming needs type_to_num_incoming_edges");
  const int V = plan->V, L = plan->L;
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  Arena ar(workspace, workspace_bytes);
  float* d_agg = ar.floats((size_t)V * d_out);
  float* d_t = ar.floats((size_t)V * L * d_out);
  float* pre = nullptr;
  float* t_fwd = nullptr;
  if (activation == RGNN_ACT_GELU) {   // gelu' needs the pre-activation: recompute it (T = H.W, agg = segment reduce)
    pre = ar.floats((size_t)V * d_out);
    t_fwd = ar.floats((size_t)V * L * d_out);
  }
  float* gw_scratch = nullptr;
  if (grad_edge_weights) gw_scratch = ar.floats(gemm_tn_scratch_floats(d_in, L * d_out, V));
  RGNN_PROPAGATE(check_ws(ar, "rgcn_backward"));

  if (pre != nullptr) {
    RGNN_PROPAGATE(gemm_shared_a(ar, h, V, d_in, edge_weights, L, d_out, d_out, t_fwd, RGNN_ACT_LINEAR, stream));
    SegParams f;
    seg_from_plan(f, plan);
    f.D = d_out; f.table = t_fwd; f.stride_idx = (long)L * d_out; f.stride_type = d_out;
    f.num_incoming = normalize ? num_incoming : nullptr;
    f.agg = aggregation; f.out = pre; f.ld_out = d_out;
    RGNN_PROPAGATE(launch_seg_reduce(f, stream));
  }
  RGNN_PROPAGATE(launch_act_backward(grad_out, out, pre, V, d_out, activation, aggregation, plan->seg_off, d_agg, stream));
  {
    SegParams r;   // reverse index: segment = (source u, type l); gathered row = d_agg[original target]
    r.V = V * L; r.L = L; r.D = d_out;
    r.seg_off = plan->rev_seg_off; r.e_idx = plan->rev_src; r.e_type = plan->rev_type;
    r.table = d_agg; r.stride_idx = d_out; r.stride_type = 0;
    r.num_incoming = normalize ? num_incoming : nullptr; r.scale_ld = V; r.scale_by_idx = 1;
    r.heavy_list = plan->rev_heavy_list; r.heavy_count = plan->err_flag + 2;
    r.heavy_threshold = RGNN_HEAVY_SEGMENT; r.heavy_known = -1;
    r.agg = RGNN_AGG_SUM; r.out = d_t; r.ld_out = d_out;
    RGNN_PROPAGATE(launch_seg_reduce(r, stream));
  }
  if (grad_h != nullptr) {
    GemmParams g;
    g.A1 = d_t; g.lda1 = L * d_out; g.K1 = L * d_out;
    g.M = V; g.N = d_in; g.C = grad_h; g.ldc = d_in; g.ldb1 = d_out;
    g.batch_mode = BATCH_K_BLOCKS_T; g.batch = L; g.k_block = d_out;
    for (int l = 0; l < L; ++l) { g.bptr[l] = edge_weights[l]; g.bptr2[l] = nullptr; }
    RGNN_PROPAGATE(run_gemm(g, ar, stream));
  }
  if (grad_edge_weights != nullptr) {
    // dW_l = H^T . dT[:, l, :]  -- one TN contraction over the V nodes for all types (gemm_tn_wgmma.cu)
    GemmTnOut tn;
    tn.block_cols = d_out; tn.ld = d_out;
    for (int l = 0; l < L; ++l) {
      RGNN_REQUIRE(grad_edge_weights[l] != nullptr && aligned16(grad_edge_weights[l]), "rgcn_backward: grad weight %d is NULL / misaligned", l);
      tn.ptr[l] = grad_edge_weights[l];
    }
    RGNN_PROPAGATE(launch_gemm_tn(h, d_in, d_t, L * d_out, d_in, L * d_out, V, tn, gw_scratch, stream));
  }
  return RGNN_OK;
}

// models/sparse_graph_model.py:176-191: for layer_idx in range(graph_num_layers): _apply_gnn_layer(...)
extern "C" int rgnn_rgcn_stack_forward(const rgnn_plan_t* plan, const float* h, int32_t d, int32_t num_layers,
                                       const float* const* edge_weights, const float* num_incoming, int activation,
                                       int aggregation, int normalize, float* out, void* workspace,
                                       size_t workspace_bytes, void* stream_) {
  RGNN_REQUIRE(plan != nullptr && num_layers >= 1, "rgcn_stack: plan is NULL or num_layers < 1");
  RGNN_REQUIRE(edge_weights != nullptr, "rgcn_stack: edge_weights is NULL");
  // layer 2 would gather halo source rows of the intermediate buffer, which no layer of this call writes
  RGNN_REQUIRE(num_layers == 1 || plan->Vt == plan->V,
               "rgcn_stack: a plan restricted to %d of %d target rows supports num_layers == 1 only (halo rows are not updated)", plan->Vt, plan->V);
  const size_t row_bytes = align_up((size_t)plan->V * d * sizeof(float), 256);
  if (workspace == nullptr || workspace_bytes <= 2 * row_bytes) {
    set_error("rgcn_stack: workspace too small (%zu bytes given, more than %zu needed for the two inter-layer buffers)",
              workspace == nullptr ? (size_t)0 : workspace_bytes, 2 * row_bytes);
    return RGNN_E_WORKSPACE;
  }
  char* base = static_cast<char*>(workspace);
  float* buf[2] = {reinterpret_cast<float*>(base), reinterpret_cast<float*>(base + row_bytes)};
  void* inner = base + 2 * row_bytes;
  const size_t inner_bytes = workspace_bytes - 2 * row_bytes;
  const float* cur = h;
  for (int l = 0; l < num_layers; ++l) {
    float* dst = (l == num_layers - 1) ? out : buf[l & 1];
    RGNN_PROPAGATE(rgnn_rgcn_forward(plan, cur, d, d, edge_weights + (size_t)l * plan->L, num_incoming, activation,
                                     aggregation, normalize, 0, 1, dst, inner, inner_bytes, stream_));
    cur = dst;
  }
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/rgdcn.py:8-171
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_rgdcn_forward(const rgnn_plan_t* plan, const float* h, int32_t d, int32_t num_channels,
                                  const float* const* channel_weights, int use_full_state, const float* num_incoming,
                                  int activation, int aggregation, int normalize, int num_timesteps, float* out,
                                  void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d, d, out, num_timesteps, "rgdcn"));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));
  RGNN_PROPAGATE(check_act(activation, "rgdcn"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgdcn"));
  RGNN_REQUIRE(channel_weights != nullptr, "rgdcn: channel_weights is NULL");
  RGNN_REQUIRE(num_channels >= 1 && num_channels <= RGNN_MAX_EDGE_TYPES && (d % num_channels) == 0,
               "rgdcn: num_channels %d must divide the state dim %d (and be <= %d)", num_channels, d, RGNN_MAX_EDGE_TYPES);
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "rgdcn: normalize_by_num_incoming needs type_to_num_incoming_edges");
  const int V = plan->V, Vt = plan->Vt, L = plan->L, C = num_channels, K = d / num_channels;
  RGNN_REQUIRE(K >= 4 && (K & (K - 1)) == 0 && K <= 128, "rgdcn: channel_dim %d must be a power of two in [4, 128]", K);
  for (int i = 0; i < L * C; ++i)
    RGNN_REQUIRE(channel_weights[i] != nullptr && aligned16(channel_weights[i]), "rgdcn: channel weight %d is NULL / misaligned", i);
  Arena ar(workspace, workspace_bytes);
  float* wdyn = ar.floats((size_t)Vt * L * d * K);   // the dynamic kernels depend on the target: wanted target rows only
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * d); buf[1] = ar.floats((size_t)V * d); }
  RGNN_PROPAGATE(check_ws(ar, "rgdcn"));
  const float* cur = h;
  for (int t = 0; t < num_timesteps; ++t) {
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    // W[v, l, c] = act(F_{l,c} . input_v) reshaped [K, K]  (:139-148; the Dense carries the layer's activation, :101-103)
    for (int l = 0; l < L; ++l) {
      GemmParams g;
      g.A1 = cur; g.lda1 = d; g.M = Vt; g.N = K * K; g.ldb1 = K * K;
      g.C = wdyn + (size_t)l * d * K; g.ldc = L * d * K;
      g.act = activation; g.batch = C;
      for (int c = 0; c < C; ++c) { g.bptr[c] = channel_weights[l * C + c]; g.bptr2[c] = nullptr; }
      if (use_full_state) { g.K1 = d; g.batch_mode = BATCH_SHARED_A; }       // input = the whole state h_v
      else { g.K1 = K; g.batch_mode = BATCH_COL_BLOCKS; }                    // input = the channel's slice h_v[c]
      RGNN_PROPAGATE(run_gemm(g, ar, stream));
    }
    RgdcnParams r;
    r.V = Vt; r.L = L; r.D = d; r.K = K;
    r.seg_off = plan->seg_off; r.e_src = plan->e_src; r.e_type = plan->e_type;
    r.h = cur; r.wdyn = wdyn; r.num_incoming = normalize ? num_incoming : nullptr; r.scale_ld = V;
    r.agg = aggregation; r.act_out = activation; r.out = dst;
    RGNN_PROPAGATE(launch_rgdcn_edges(r, stream));
    cur = dst;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_rgdcn_layer (sum / mean / sqrt_n): what tf.gradients produces for gnns/rgdcn.py:116-165.
// No forward state is kept and nothing per edge is built (rgdcn_backward.cu has the math of the edge kernel):
//   P = x . F_{l,c} (wgmma GEMM, no activation: the Vt wanted target rows)
//   per target: a, delta, dS [V, L, D] (rows >= Vt zero) and dP over P                     (rgdcn_bwd_target_kernel)
//   d_h = sum_l (sum_{(u->v) in A_l} dS[v, l])  (reverse-index segment reduce, then the types in order)
//         + dP . F^T on the Vt target rows (transposed-image GEMM)
//   dF_{l,c} = x^T . dP[:, l, c] (split-K TN GEMM; tied: one dF_l = sum over c)
// Layout of P: full state keeps the forward's [Vt, L, C, K*K], so the d_h term is a BATCH_K_BLOCKS_T GEMM over the L C
// kernels and dF one TN GEMM with a K*K column block per kernel (both in chunks of RGNN_MAX_EDGE_TYPES kernels).  Per channel
// it is [Vt, C, L, K*K]: the L kernels of a channel are adjacent, so d_h[:, c] is a BATCH_K_BLOCKS_T GEMM per channel, dF of
// channel c one TN GEMM over h[:, c], and the tied dF_l one TN GEMM over h viewed as [Vt C, K] rows.  The d_h GEMMs contract
// at most 1,024 columns of dP per launch (see below).
extern "C" int rgnn_rgdcn_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d, int32_t num_channels,
                                   const float* const* channel_weights, int use_full_state, int tie_channel_weights,
                                   const float* num_incoming, int activation, int aggregation, int normalize,
                                   const float* grad_out, float* grad_h, float* const* grad_channel_weights,
                                   void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr, "rgdcn_backward: plan is NULL");
  RGNN_REQUIRE(h != nullptr, "rgdcn_backward: node_embeddings is NULL");
  RGNN_REQUIRE(grad_out != nullptr, "rgdcn_backward: grad_out is NULL");
  RGNN_REQUIRE(channel_weights != nullptr, "rgdcn_backward: channel_weights is NULL");
  RGNN_REQUIRE(d > 0 && (d % 4) == 0, "rgdcn_backward: the state dim d = %d must be a positive multiple of 4", d);
  if (d > RGNN_MAX_STATE_DIM) {
    set_error("rgdcn_backward: the state dim d = %d > %d is not supported in this build", d, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_PROPAGATE(check_act(activation, "rgdcn_backward"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgdcn_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("rgdcn_backward: the gradient of 'max' aggregation is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_REQUIRE(num_channels >= 1 && num_channels <= RGNN_MAX_EDGE_TYPES && (d % num_channels) == 0,
               "rgdcn_backward: num_channels %d must divide the state dim %d (and be <= %d)", num_channels, d, RGNN_MAX_EDGE_TYPES);
  const int V = plan->V, Vt = plan->Vt, L = plan->L, C = num_channels, K = d / num_channels, KK = K * K, LC = L * C;
  const bool full = use_full_state != 0, tied = tie_channel_weights != 0;
  RGNN_REQUIRE(K >= 4 && (K & (K - 1)) == 0 && K <= 128, "rgdcn_backward: channel_dim %d must be a power of two in [4, 128]", K);
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "rgdcn_backward: normalize_by_num_incoming needs num_incoming");
  for (int i = 0; i < LC; ++i)
    RGNN_REQUIRE(channel_weights[i] != nullptr && aligned16(channel_weights[i]), "rgdcn_backward: channel weight %d is NULL / misaligned", i);
  if (tied)
    for (int i = 0; i < LC; ++i)
      RGNN_REQUIRE(channel_weights[i] == channel_weights[i - i % C],
                   "rgdcn_backward: tie_channel_weights = 1 needs one kernel per edge type, but channel_weights[%d] != channel_weights[%d]",
                   i, i - i % C);
  RGNN_REQUIRE(aligned16(h) && aligned16(grad_out), "rgdcn_backward: node_embeddings / grad_out must be 16-byte aligned");
  RGNN_REQUIRE(aligned16(grad_h), "rgdcn_backward: grad_node_embeddings must be 16-byte aligned");
  RGNN_REQUIRE(grad_h == nullptr || (grad_h != h && grad_h != grad_out),
               "rgdcn_backward: grad_node_embeddings must not alias node_embeddings or grad_out");
  float* const* gw = grad_channel_weights;
  if (gw != nullptr) {
    for (int i = 0; i < LC; ++i)
      RGNN_REQUIRE(gw[i] != nullptr && aligned16(gw[i]), "rgdcn_backward: grad channel weight %d is NULL / misaligned", i);
    std::pair<float*, int> seen[RGNN_MAX_EDGE_TYPES * RGNN_MAX_EDGE_TYPES];   // the distinct kernels' gradients
    int n = 0;
    for (int i = 0; i < LC; ++i) {
      if (tied && i % C != 0) {
        RGNN_REQUIRE(gw[i] == gw[i - i % C],
                     "rgdcn_backward: tie_channel_weights = 1 needs one gradient per edge type, but grad_channel_weights[%d] != grad_channel_weights[%d]",
                     i, i - i % C);
        continue;
      }
      seen[n++] = {gw[i], i};
    }
    std::sort(seen, seen + n);
    for (int i = 1; i < n; ++i)
      RGNN_REQUIRE(seen[i].first != seen[i - 1].first, "rgdcn_backward: grad_channel_weights[%d] and grad_channel_weights[%d] alias",
                   std::min(seen[i - 1].second, seen[i].second), std::max(seen[i - 1].second, seen[i].second));
  }

  // the P recompute: launch i is chunk i of RGNN_MAX_EDGE_TYPES kernels (full state) or channel i
  const int n_dense = full ? (LC + RGNN_MAX_EDGE_TYPES - 1) / RGNN_MAX_EDGE_TYPES : C;
  Arena ar(workspace, workspace_bytes);
  float* P = ar.floats((size_t)Vt * LC * KK);
  float* dS = ar.floats((size_t)V * L * d);
  float* dQ = grad_h != nullptr ? ar.floats((size_t)V * L * d) : nullptr;
  float* kin = grad_h != nullptr ? ar.floats((size_t)Vt * d) : nullptr;   // the kernel-input term of d_h
  float* psum = (gw != nullptr && full && tied) ? ar.floats((size_t)Vt * L * KK) : nullptr;
  auto chunk = [&](int i, int& z0, int& nz) { z0 = i * RGNN_MAX_EDGE_TYPES; nz = std::min(RGNN_MAX_EDGE_TYPES, LC - z0); };
  auto fwd_p = [&](int i) {   // P = x . F (no activation)
    GemmParams g;
    g.M = Vt; g.N = KK; g.ldb1 = KK; g.batch_mode = BATCH_SHARED_A;
    if (full) {
      int z0, nz;
      chunk(i, z0, nz);
      g.A1 = h; g.lda1 = d; g.K1 = d; g.batch = nz; g.C = P + (size_t)z0 * KK; g.ldc = LC * KK;
      for (int z = 0; z < nz; ++z) { g.bptr[z] = channel_weights[z0 + z]; g.bptr2[z] = nullptr; }
    } else {
      g.A1 = h + (size_t)i * K; g.lda1 = d; g.K1 = K; g.batch = L; g.C = P + (size_t)i * L * KK; g.ldc = LC * KK;
      for (int l = 0; l < L; ++l) { g.bptr[l] = channel_weights[l * C + i]; g.bptr2[l] = nullptr; }
    }
    return g;
  };
  // kin = dP . F^T, contracted piece by piece: the tensor cores' fp32 accumulation loses accuracy along a long contraction
  // (L K^2 = 65,536 at K = 128 gave 1e-4 relative error in one launch), so each launch contracts at most
  // RGDCN_BWD_MAX_CHAIN columns of dP and the pieces are added into d_h in order.  A piece is the whole blocks z0 .. z0 + nz - 1
  // (kc = K*K) or the columns [j0, j0 + kc) of block z0 (nz = 1); a block is one kernel F_{l,c} (per channel: the L kernels
  // of one channel, z = l).
  constexpr int RGDCN_BWD_MAX_CHAIN = 1024;
  struct Piece { int z0, nz, j0, kc; };
  std::vector<Piece> pieces;
  {
    const int nblk = full ? LC : L;
    if (KK <= RGDCN_BWD_MAX_CHAIN) {
      const int per = std::min(RGDCN_BWD_MAX_CHAIN / KK, (int)RGNN_MAX_EDGE_TYPES);
      for (int z0 = 0; z0 < nblk; z0 += per) pieces.push_back({z0, std::min(per, nblk - z0), 0, KK});
    } else {
      for (int z = 0; z < nblk; ++z)
        for (int j0 = 0; j0 < KK; j0 += RGDCN_BWD_MAX_CHAIN) pieces.push_back({z, 1, j0, RGDCN_BWD_MAX_CHAIN});
    }
  }
  auto bwd_h = [&](const Piece& pc, int c) {   // full state: c unused
    GemmParams g;
    g.M = Vt; g.ldb1 = KK; g.k_block = pc.kc; g.K1 = pc.nz * pc.kc; g.batch = pc.nz; g.batch_mode = BATCH_K_BLOCKS_T;
    g.lda1 = LC * KK; g.ldc = d;
    if (full) {
      g.A1 = P + (size_t)pc.z0 * KK + pc.j0; g.N = d; g.C = kin;
      for (int z = 0; z < pc.nz; ++z) { g.bptr[z] = channel_weights[pc.z0 + z] + pc.j0; g.bptr2[z] = nullptr; }
    } else {
      g.A1 = P + ((size_t)c * L + pc.z0) * KK + pc.j0; g.N = K; g.C = kin + (size_t)c * K;
      for (int z = 0; z < pc.nz; ++z) { g.bptr[z] = channel_weights[(pc.z0 + z) * C + c] + pc.j0; g.bptr2[z] = nullptr; }
    }
    return g;
  };
  float* tn_scratch = nullptr;
  if (gw != nullptr) {
    size_t n = 0;
    if (full && tied) n = gemm_tn_scratch_floats(d, L * KK, Vt);
    else if (full) for (int i = 0; i < n_dense; ++i) { int z0, nz; chunk(i, z0, nz); n = std::max(n, gemm_tn_scratch_floats(d, nz * KK, Vt)); }
    else n = gemm_tn_scratch_floats(K, L * KK, tied ? Vt * C : Vt);
    tn_scratch = ar.floats(n);
  }
  size_t pack = 0;
  if (Vt > 0)
    for (int i = 0; i < n_dense; ++i) pack = std::max(pack, gemm_tc_pack_bytes(fwd_p(i)));
  if (Vt > 0 && grad_h != nullptr)
    for (const Piece& pc : pieces)
      for (int c = 0; c < (full ? 1 : C); ++c) pack = std::max(pack, gemm_tc_pack_bytes(bwd_h(pc, c)));
  {
    const size_t mark = ar.used;
    ar.floats(pack / sizeof(float));
    RGNN_PROPAGATE(check_ws(ar, "rgdcn_backward"));
    ar.used = mark;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));   // the edge kernel gathers halo source rows

  if (Vt > 0)
    for (int i = 0; i < n_dense; ++i) RGNN_PROPAGATE(run_gemm(fwd_p(i), ar, stream));
  RgdcnBwdParams r;
  r.V = V; r.Vt = Vt; r.L = L; r.D = d; r.K = K; r.C = C; r.act = activation; r.agg = aggregation;
  r.st_type = full ? C : 1; r.st_chan = full ? 1 : L;
  r.seg_off = plan->seg_off; r.e_src = plan->e_src; r.e_type = plan->e_type;
  r.h = h; r.grad_out = grad_out; r.num_incoming = normalize ? num_incoming : nullptr; r.scale_ld = V;
  r.P = P; r.dS = dS;
  RGNN_PROPAGATE(launch_rgdcn_bwd_target(r, stream));

  if (grad_h != nullptr) {
    SegParams s;   // reverse index: segment = (source u, type l); gathered row = dS[original target, l]
    s.V = V * L; s.L = L; s.D = d;
    s.seg_off = plan->rev_seg_off; s.e_idx = plan->rev_src; s.e_type = plan->rev_type;
    s.table = dS; s.stride_idx = (long)L * d; s.stride_type = d;
    s.heavy_list = plan->rev_heavy_list; s.heavy_count = plan->err_flag + 2;
    s.heavy_threshold = RGNN_HEAVY_SEGMENT; s.heavy_known = -1;
    s.agg = RGNN_AGG_SUM; s.out = dQ; s.ld_out = d;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    RGNN_PROPAGATE(launch_rgin_type_sum(dQ, V, L, d, grad_h, stream));
    if (Vt > 0)
      for (const Piece& pc : pieces) {   // in order
        for (int c = 0; c < (full ? 1 : C); ++c) RGNN_PROPAGATE(run_gemm(bwd_h(pc, c), ar, stream));
        RGNN_PROPAGATE(launch_add_rows(grad_h, kin, (long)Vt * d, stream));
      }
  }
  if (gw != nullptr) {
    GemmTnOut tn;
    tn.block_cols = KK; tn.ld = KK;
    if (full && tied) {
      RGNN_PROPAGATE(launch_rgdcn_chan_sum(P, (long)Vt * L, C, KK, psum, stream));
      for (int l = 0; l < L; ++l) tn.ptr[l] = gw[l * C];
      RGNN_PROPAGATE(launch_gemm_tn(h, d, psum, L * KK, d, L * KK, Vt, tn, tn_scratch, stream));
    } else if (full) {
      for (int i = 0; i < n_dense; ++i) {
        int z0, nz;
        chunk(i, z0, nz);
        for (int z = 0; z < nz; ++z) tn.ptr[z] = gw[z0 + z];
        RGNN_PROPAGATE(launch_gemm_tn(h, d, P + (size_t)z0 * KK, LC * KK, d, nz * KK, Vt, tn, tn_scratch, stream));
      }
    } else if (tied) {   // h as [Vt C, K] rows, dP as [Vt C, L K*K] rows
      for (int l = 0; l < L; ++l) tn.ptr[l] = gw[l * C];
      RGNN_PROPAGATE(launch_gemm_tn(h, K, P, L * KK, K, L * KK, Vt * C, tn, tn_scratch, stream));
    } else {
      for (int c = 0; c < C; ++c) {
        for (int l = 0; l < L; ++l) tn.ptr[l] = gw[l * C + c];
        RGNN_PROPAGATE(launch_gemm_tn(h + (size_t)c * K, d, P + (size_t)c * L * KK, LC * KK, K, L * KK, Vt, tn, tn_scratch, stream));
      }
    }
  }
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/ggnn.py:8-95
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_ggnn_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                 const float* const* edge_weights, const float* cell_kernel,
                                 const float* cell_recurrent_kernel, const float* cell_bias, int cell_kind,
                                 int activation, int aggregation, int num_timesteps, float* out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "ggnn"));
  RGNN_PROPAGATE(check_act(activation, "ggnn"));
  RGNN_PROPAGATE(check_agg(aggregation, "ggnn"));
  RGNN_REQUIRE(d_in == d_out, "ggnn: the recurrent cell needs state_dim == input dim (d_in=%d, d_out=%d)", d_in, d_out);
  if (cell_kind != RGNN_CELL_RNN && cell_kind != RGNN_CELL_GRU) {
    set_error("Unknown RNN cell type code %d.", cell_kind);                   // utils/utils.py:20
    return RGNN_E_INVALID;
  }
  RGNN_REQUIRE(edge_weights && cell_kernel && cell_recurrent_kernel && cell_bias, "ggnn: NULL weight pointer");
  RGNN_REQUIRE(aligned16(cell_kernel) && aligned16(cell_recurrent_kernel), "ggnn: cell kernels must be 16-byte aligned");
  const int V = plan->V, L = plan->L, D = d_out;
  for (int l = 0; l < L; ++l) RGNN_REQUIRE(edge_weights[l] != nullptr, "ggnn: edge weight %d is NULL", l);
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);
  float* m = ar.floats((size_t)V * D);
  const int slab_max = RGNN_WAVE_SMS * 128;                                   // GRU rows per slab: one wave of 128-row tiles
  const int slab = V < slab_max ? (V > 0 ? V : 1) : slab_max;
  float* z = ar.floats((size_t)slab * D);
  float* rh = ar.floats((size_t)slab * D);
  float* buf[2] = {ar.floats((size_t)V * D), ar.floats((size_t)V * D)};
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, D);
  RGNN_PROPAGATE(check_ws(ar, "ggnn"));

  const float* cur = h;
  for (int t = 0; t < num_timesteps; ++t) {                                   // ggnn.py:71
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    SegParams s;
    seg_from_plan(s, plan);
    s.D = D;
    RGNN_PROPAGATE(transform_sources(plan, ar, cur, D, D, edge_weights, T, stream, s));   // ggnn.py:80-82
    s.agg = aggregation; s.out = m; s.ld_out = D; s.heavy_scratch = heavy.heavy_scratch;   // ggnn.py:87-90
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    GemmParams g;
    g.A1 = m; g.lda1 = D; g.K1 = D;
    g.M = plan->Vt; g.bias = cell_bias;   // the cell runs on the wanted target rows only
    if (cell_kind == RGNN_CELL_RNN) {                                         // SimpleRNNCell: act(x.W + b + h.U)
      g.A2 = cur; g.lda2 = D; g.K2 = D;
      g.B1 = cell_kernel; g.ldb1 = D; g.B2 = cell_recurrent_kernel; g.ldb2 = D;
      g.N = D; g.C = dst; g.ldc = D; g.epi = EPI_STORE; g.act = activation;
      RGNN_PROPAGATE(run_gemm(g, ar, stream));
    } else {                                                                  // GRUCell, gates z|r|h (A.4)
      // Two GEMMs per row SLAB: [z | r.h] = hs([m|h].[W_zr;U_zr] + b), then h' = z.h + (1-z).act([m | r.h].[W_h;U_h] + b_h).
      // z and r.h live in slab-sized scratch that every slab overwrites: with ~17k rows per slab (one wave of 128-row
      // tiles on 132 SMs) the slab's z, r.h, m, h and output rows (5 x 8.7 MB at D = 128) fit the 50 MB L2 between the two
      // kernels, and the dirty z / r.h lines are overwritten before they are evicted instead of making a round trip through HBM.
      const int Vc = plan->Vt;
      for (int r0 = 0; r0 < Vc; r0 += slab) {
        const int rows = (Vc - r0 < slab) ? Vc - r0 : slab;
        const size_t off = (size_t)r0 * D;
        GemmParams g2 = g;
        g2.A1 = m + off; g2.M = rows;
        g2.A2 = cur + off; g2.lda2 = D; g2.K2 = D;
        g2.B1 = cell_kernel; g2.ldb1 = 3 * D; g2.B2 = cell_recurrent_kernel; g2.ldb2 = 3 * D;
        g2.N = 2 * D; g2.C = z; g2.ldc = D; g2.C2 = rh; g2.ldc2 = D; g2.aux_h = cur + off; g2.ld_h = D;
        g2.epi = EPI_GRU_ZR;
        RGNN_PROPAGATE(run_gemm(g2, ar, stream));
        GemmParams o;
        o.A1 = m + off; o.lda1 = D; o.K1 = D; o.A2 = rh; o.lda2 = D; o.K2 = D;
        o.B1 = cell_kernel + 2 * D; o.ldb1 = 3 * D; o.B2 = cell_recurrent_kernel + 2 * D; o.ldb2 = 3 * D;
        o.M = rows; o.N = D; o.bias = cell_bias + 2 * D; o.C = dst + off; o.ldc = D;
        o.aux_h = cur + off; o.ld_h = D; o.aux_z = z; o.ld_z = D;
        o.epi = EPI_GRU_OUT; o.act = activation;
        RGNN_PROPAGATE(run_gemm(o, ar, stream));
      }
    }
    cur = dst;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_ggnn_layer: what tf.gradients produces for gnns/ggnn.py:76-93.  No forward state is
// kept: m and the cell's pre-activations are recomputed (ggnn_backward.cu has the element-wise math).
//   T = h . [W_0|..|W_{L-1}], m = agg T (transform_sources + segment reduce, as the forward)
//   GRU: [a_z|a_r] = [m|h] . [K_zr;R_zr] + b_zr,  rh = r h,  a_h = [m|rh] . [K_h;R_h] + b_h       (wgmma GEMM, A2 = 2nd operand)
//        da_z, da_h, e = g z;  d(rh) = da_h . R_h^T;  da_r, e += d(rh) r;  f = [da_z|da_r] . R_zr^T
//   RNN: a = [m|h] . [K;R] + b;  da = g act'(a);  f = da . R^T
//   dm = da . K^T (/ div(v); rows >= Vt are zero),  dT[u,l] = sum_{(u->v) in A_l} dm[v]   (reverse index; dT reuses T)
//   d_h = dT . [W_l]^T (V rows), then rows < Vt += e + f          d_W_l = h^T . dT[:, l, :]
//   d_K = m^T . da,  d_R = h^T . [da_z|da_r] | rh^T . da_h  (RNN: h^T . da),  d_b = column sums of da (CTA partials, fixed order)
extern "C" int rgnn_ggnn_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d, const float* const* edge_weights,
                                  const float* cell_kernel, const float* cell_recurrent_kernel, const float* cell_bias,
                                  int cell_kind, int activation, int aggregation, const float* grad_out, float* grad_h,
                                  float* const* grad_edge_weights, float* grad_cell_kernel,
                                  float* grad_cell_recurrent_kernel, float* grad_cell_bias, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr, "ggnn_backward: plan is NULL");
  RGNN_REQUIRE(h != nullptr, "ggnn_backward: node_embeddings is NULL");
  RGNN_REQUIRE(edge_weights != nullptr, "ggnn_backward: edge_weights is NULL");
  RGNN_REQUIRE(cell_kernel != nullptr, "ggnn_backward: cell_kernel is NULL");
  RGNN_REQUIRE(cell_recurrent_kernel != nullptr, "ggnn_backward: cell_recurrent_kernel is NULL");
  RGNN_REQUIRE(cell_bias != nullptr, "ggnn_backward: cell_bias is NULL");
  RGNN_REQUIRE(grad_out != nullptr, "ggnn_backward: grad_out is NULL");
  RGNN_REQUIRE(d > 0 && (d % 4) == 0, "ggnn_backward: state dim d must be a positive multiple of 4 (d=%d)", d);
  RGNN_REQUIRE(cell_kind == RGNN_CELL_RNN || cell_kind == RGNN_CELL_GRU, "ggnn_backward: Unknown RNN cell type code %d", cell_kind);
  RGNN_PROPAGATE(check_act(activation, "ggnn_backward"));
  RGNN_PROPAGATE(check_agg(aggregation, "ggnn_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("ggnn_backward: the gradient of 'max' aggregation is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_REQUIRE(aligned16(h) && aligned16(grad_out), "ggnn_backward: node_embeddings / grad_out must be 16-byte aligned");
  RGNN_REQUIRE(aligned16(cell_kernel) && aligned16(cell_recurrent_kernel) && aligned16(cell_bias),
               "ggnn_backward: cell_kernel / cell_recurrent_kernel / cell_bias must be 16-byte aligned");
  RGNN_REQUIRE(aligned16(grad_h) && aligned16(grad_cell_kernel) && aligned16(grad_cell_recurrent_kernel) && aligned16(grad_cell_bias),
               "ggnn_backward: grad_node_embeddings / grad_cell_kernel / grad_cell_recurrent_kernel / grad_cell_bias must be 16-byte aligned");
  RGNN_REQUIRE(grad_h == nullptr || (grad_h != h && grad_h != grad_out),
               "ggnn_backward: grad_node_embeddings must not alias node_embeddings or grad_out");
  const int V = plan->V, Vt = plan->Vt, L = plan->L, D = d;
  const bool gru = cell_kind == RGNN_CELL_GRU;
  const int G = gru ? 3 : 1;   // gates
  for (int l = 0; l < L; ++l) {
    RGNN_REQUIRE(edge_weights[l] != nullptr, "ggnn_backward: edge weight %d is NULL", l);
    RGNN_REQUIRE(grad_edge_weights == nullptr || (grad_edge_weights[l] != nullptr && aligned16(grad_edge_weights[l])),
                 "ggnn_backward: grad edge weight %d is NULL / misaligned", l);
  }

  // every carve-out and the largest weight-image scratch of the dense contractions, before anything is enqueued
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);                   // T, then dT
  float* m = ar.floats((size_t)Vt * D);
  float* dm = ar.floats((size_t)V * D);
  float* a = ar.floats((size_t)Vt * G * D);                  // pre-activations
  float* da = gru ? ar.floats((size_t)Vt * G * D) : a;       // the RNN backward overwrites a with da
  float* rh = gru ? ar.floats((size_t)Vt * D) : nullptr;
  float* f = ar.floats((size_t)Vt * D);                      // GRU: d(rh), then the R_zr term of d_h; RNN: da . R^T
  float* e = (gru && grad_h != nullptr) ? ar.floats((size_t)Vt * D) : nullptr;
  float* b_part = grad_cell_bias != nullptr ? ar.floats((size_t)ggnn_colsum_blocks(Vt) * G * D + 4) : nullptr;
  float* tn_scratch = nullptr;
  if (grad_edge_weights != nullptr || grad_cell_kernel != nullptr || grad_cell_recurrent_kernel != nullptr) {
    size_t n = gemm_tn_scratch_floats(D, G * D, Vt);
    n = std::max(n, gemm_tn_scratch_floats(D, L * D, V));
    if (gru) n = std::max(n, std::max(gemm_tn_scratch_floats(D, 2 * D, Vt), gemm_tn_scratch_floats(D, D, Vt)));
    tn_scratch = ar.floats(n);
  }
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, D);

  // the dense contractions
  GemmParams gA, gAh, gRh, gM, gF, gH;
  gA.A1 = m; gA.lda1 = D; gA.K1 = D; gA.A2 = h; gA.lda2 = D; gA.K2 = D;           // [a_z|a_r] (GRU) / a (RNN)
  gA.B1 = cell_kernel; gA.ldb1 = G * D; gA.B2 = cell_recurrent_kernel; gA.ldb2 = G * D;
  gA.M = Vt; gA.N = gru ? 2 * D : D; gA.bias = cell_bias; gA.C = a; gA.ldc = G * D;
  gAh = gA;                                                                      // a_h = [m|rh] . [K_h;R_h] + b_h
  gAh.A2 = rh; gAh.B1 = cell_kernel + 2 * D; gAh.B2 = cell_recurrent_kernel + 2 * D; gAh.N = D; gAh.bias = cell_bias + 2 * D;
  gAh.C = a + 2 * D;
  gRh.A1 = da + 2 * D; gRh.lda1 = 3 * D; gRh.K1 = D; gRh.M = Vt; gRh.N = D; gRh.C = f; gRh.ldc = D;   // d(rh) = da_h . R_h^T
  gRh.batch_mode = BATCH_K_BLOCKS_T; gRh.batch = 1; gRh.k_block = D; gRh.bptr[0] = cell_recurrent_kernel + 2 * D; gRh.ldb1 = 3 * D;
  gRh.bptr2[0] = nullptr;
  gM.A1 = da; gM.lda1 = G * D; gM.K1 = G * D; gM.M = Vt; gM.N = D; gM.C = dm; gM.ldc = D;          // dm = da . K^T
  gM.batch_mode = BATCH_K_BLOCKS_T; gM.batch = 1; gM.k_block = G * D; gM.bptr[0] = cell_kernel; gM.ldb1 = G * D;
  gM.bptr2[0] = nullptr;
  gF = gM;                                                       // f = [da_z|da_r] . R_zr^T (GRU) / da . R^T (RNN)
  gF.K1 = gF.k_block = gru ? 2 * D : D; gF.bptr[0] = cell_recurrent_kernel; gF.C = f;
  gH.A1 = T; gH.lda1 = L * D; gH.K1 = L * D; gH.M = V; gH.N = D; gH.C = grad_h; gH.ldc = D; gH.ldb1 = D;   // dT . [W_l]^T
  gH.batch_mode = BATCH_K_BLOCKS_T; gH.batch = L; gH.k_block = D;
  for (int l = 0; l < L; ++l) { gH.bptr[l] = edge_weights[l]; gH.bptr2[l] = nullptr; }
  size_t pack = transform_sources_pack_bytes(plan, D, D);
  if (Vt > 0) {
    pack = std::max(pack, std::max(gemm_tc_pack_bytes(gA), gemm_tc_pack_bytes(gM)));
    if (gru) pack = std::max(pack, std::max(gemm_tc_pack_bytes(gAh), gemm_tc_pack_bytes(gRh)));
    if (grad_h != nullptr) pack = std::max(pack, gemm_tc_pack_bytes(gF));
  }
  if (grad_h != nullptr && V > 0) pack = std::max(pack, gemm_tc_pack_bytes(gH));
  {
    const size_t mark = ar.used;
    ar.floats(pack / sizeof(float));
    RGNN_PROPAGATE(check_ws(ar, "ggnn_backward"));
    ar.used = mark;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));

  // forward: m (transform_sources waits for a pending halo exchange), then the cell's pre-activations
  {
    SegParams s;
    seg_from_plan(s, plan);
    s.D = D;
    RGNN_PROPAGATE(transform_sources(plan, ar, h, D, D, edge_weights, T, stream, s));
    s.agg = aggregation; s.out = m; s.ld_out = D; s.heavy_scratch = heavy.heavy_scratch;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
  }
  GgnnCellBwdParams cp;
  cp.rows = Vt; cp.D = D; cp.act = activation; cp.grad_out = grad_out; cp.h = h; cp.a = a; cp.da = da; cp.drh = f; cp.e = e;
  if (Vt > 0) {
    RGNN_PROPAGATE(run_gemm(gA, ar, stream));
    if (gru) {
      RGNN_PROPAGATE(launch_ggnn_gru_rh(a, h, Vt, D, rh, stream));
      RGNN_PROPAGATE(run_gemm(gAh, ar, stream));
      // the cell backward
      RGNN_PROPAGATE(launch_ggnn_cell_backward(cp, cell_kind, 0, stream));
      RGNN_PROPAGATE(run_gemm(gRh, ar, stream));
      RGNN_PROPAGATE(launch_ggnn_cell_backward(cp, cell_kind, 1, stream));
    } else {
      RGNN_PROPAGATE(launch_ggnn_cell_backward(cp, cell_kind, 0, stream));
    }
    RGNN_PROPAGATE(run_gemm(gM, ar, stream));
  }
  // the edge stage: dT[u, l] = sum over the edges (u -> v) of type l of dm[v]; dT overwrites T
  RGNN_PROPAGATE(launch_ggnn_dm_finish(dm, V, Vt, D, aggregation, plan->seg_off, stream));
  {
    SegParams r;   // reverse index: segment = (source u, type l); gathered row = dm[original target]
    r.V = V * L; r.L = L; r.D = D;
    r.seg_off = plan->rev_seg_off; r.e_idx = plan->rev_src; r.e_type = plan->rev_type;
    r.table = dm; r.stride_idx = D; r.stride_type = 0;
    r.heavy_list = plan->rev_heavy_list; r.heavy_count = plan->err_flag + 2;
    r.heavy_threshold = RGNN_HEAVY_SEGMENT; r.heavy_known = -1;
    r.agg = RGNN_AGG_SUM; r.out = T; r.ld_out = D;
    RGNN_PROPAGATE(launch_seg_reduce(r, stream));
  }

  // the outputs, each written once
  if (grad_edge_weights != nullptr) {
    GemmTnOut tn;
    tn.block_cols = D; tn.ld = D;
    for (int l = 0; l < L; ++l) tn.ptr[l] = grad_edge_weights[l];
    RGNN_PROPAGATE(launch_gemm_tn(h, D, T, L * D, D, L * D, V, tn, tn_scratch, stream));
  }
  if (grad_cell_kernel != nullptr) {
    GemmTnOut tn;
    tn.block_cols = G * D; tn.ld = G * D; tn.ptr[0] = grad_cell_kernel;
    RGNN_PROPAGATE(launch_gemm_tn(m, D, da, G * D, D, G * D, Vt, tn, tn_scratch, stream));
  }
  if (grad_cell_recurrent_kernel != nullptr) {
    GemmTnOut tn;
    tn.ld = G * D;
    if (gru) {
      tn.block_cols = 2 * D; tn.ptr[0] = grad_cell_recurrent_kernel;
      RGNN_PROPAGATE(launch_gemm_tn(h, D, da, 3 * D, D, 2 * D, Vt, tn, tn_scratch, stream));
      tn.block_cols = D; tn.ptr[0] = grad_cell_recurrent_kernel + 2 * D;
      RGNN_PROPAGATE(launch_gemm_tn(rh, D, da + 2 * D, 3 * D, D, D, Vt, tn, tn_scratch, stream));
    } else {
      tn.block_cols = D; tn.ptr[0] = grad_cell_recurrent_kernel;
      RGNN_PROPAGATE(launch_gemm_tn(h, D, da, D, D, D, Vt, tn, tn_scratch, stream));
    }
  }
  if (grad_cell_bias != nullptr) RGNN_PROPAGATE(launch_ggnn_bias_grad(da, Vt, G * D, b_part, grad_cell_bias, stream));
  if (grad_h != nullptr) {
    if (V > 0) RGNN_PROPAGATE(run_gemm(gH, ar, stream));
    if (Vt > 0) {
      RGNN_PROPAGATE(run_gemm(gF, ar, stream));
      RGNN_PROPAGATE(launch_ggnn_add_cell_grad(grad_h, gru ? e : f, gru ? f : nullptr, (long)Vt * D, stream));
    }
  }
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/rgat.py:9-141
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_rgat_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                 const float* const* edge_weights, const float* const* attention, int num_heads,
                                 int activation, int num_timesteps, float* out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "rgat"));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));
  RGNN_PROPAGATE(check_act(activation, "rgat"));
  RGNN_REQUIRE(edge_weights != nullptr && attention != nullptr, "rgat: NULL weight table");
  RGNN_REQUIRE(num_heads >= 1 && (d_out % num_heads) == 0, "rgat: state_dim %d not divisible by num_heads %d", d_out, num_heads);
  const int V = plan->V, L = plan->L, D = d_out, K = num_heads;
  AttnTable at;
  for (int l = 0; l < L; ++l) {
    RGNN_REQUIRE(edge_weights[l] != nullptr && attention[l] != nullptr && aligned16(attention[l]), "rgat: weight %d is NULL / misaligned", l);
    at.att[l] = attention[l];
  }
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);
  // per-edge logits: computed inside the edge kernel when a head's dh/4 lanes form a power-of-two group inside one warp
  const int dh = D / K, lph = dh / 4;
  const bool fused_scores = (dh % 4) == 0 && lph >= 1 && lph <= 32 && (lph & (lph - 1)) == 0;
  float* ssrc = fused_scores ? nullptr : ar.floats((size_t)V * L * K);
  float* stgt = fused_scores ? nullptr : ar.floats((size_t)V * L * K);
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * D); buf[1] = ar.floats((size_t)V * D); }
  RGNN_PROPAGATE(check_ws(ar, "rgat"));

  const float* cur = h;
  int din = d_in;
  for (int t = 0; t < num_timesteps; ++t) {                                   // rgat.py:83
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    RGNN_PROPAGATE(gemm_shared_a(ar, cur, V, din, edge_weights, L, D, D, T, RGNN_ACT_LINEAR, stream));   // rgat.py:95-96
    if (!fused_scores) RGNN_PROPAGATE(launch_rgat_scores(T, V, L, D, K, at, ssrc, stgt, stream));   // rgat.py:106-115 (per node)
    RgatParams r;
    r.V = plan->Vt; r.L = L; r.D = D; r.K = K; r.att = at;                  // T covers every source row, the softmax only the wanted targets
    r.seg_off = plan->seg_off; r.e_src = plan->e_src; r.e_type = plan->e_type;
    r.table = T; r.s_src = ssrc; r.s_tgt = stgt; r.act_out = activation; r.out = dst;
    RGNN_PROPAGATE(launch_seg_rgat(r, stream));                                                      // rgat.py:120-138
    cur = dst; din = D;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_rgat_layer: what tf.gradients produces for gnns/rgat.py:83-139.  No forward state is
// kept: the tables are recomputed (rgat_backward.cu has the math).
//   T = h . [W_0|..|W_{L-1}] (V rows), s_src / s_tgt = per-head scores of T (rgat_scores_kernel)
//   target side (CSR by target): softmax statistics, d_o = act'(o) grad_out, c, D_tgt      source side (reverse index): dT, D_src
//   d_att_l = [sum_u D_src T | sum_{v<Vt} D_tgt T] per head           per-CTA partials, fixed-order sum
//   d_h = dT . [W_l]^T (V rows)   transposed-image GEMM;   d_W_l = h^T . dT[:, l, :]   TN GEMM, split-K, deterministic
extern "C" int rgnn_rgat_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d_in, int32_t d_out,
                                  const float* const* edge_weights, const float* const* attention, int num_heads, int activation,
                                  const float* grad_out, float* grad_h, float* const* grad_edge_weights,
                                  float* const* grad_attention, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr, "rgat_backward: plan is NULL");
  RGNN_REQUIRE(h != nullptr, "rgat_backward: node_embeddings is NULL");
  RGNN_REQUIRE(edge_weights != nullptr, "rgat_backward: edge_weights is NULL");
  RGNN_REQUIRE(attention != nullptr, "rgat_backward: attention is NULL");
  RGNN_REQUIRE(grad_out != nullptr, "rgat_backward: grad_out is NULL");
  RGNN_REQUIRE(d_in > 0 && d_out > 0 && (d_in % 4) == 0 && (d_out % 4) == 0,
               "rgat_backward: d_in / d_out must be positive multiples of 4 (d_in=%d, d_out=%d)", d_in, d_out);
  if (d_out > RGNN_MAX_STATE_DIM) {
    set_error("rgat_backward: d_out %d > %d (a warp holds a whole row) is not supported", d_out, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_REQUIRE(num_heads >= 1 && (d_out % num_heads) == 0, "rgat_backward: num_heads %d does not divide d_out %d", num_heads, d_out);
  if (((d_out / num_heads) % 4) != 0) {
    set_error("rgat_backward: per-head dim %d (d_out %d / num_heads %d) must be a multiple of 4", d_out / num_heads, d_out, num_heads);
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_PROPAGATE(check_act(activation, "rgat_backward"));
  RGNN_REQUIRE(aligned16(h) && aligned16(grad_out) && aligned16(grad_h),
               "rgat_backward: node_embeddings / grad_out / grad_node_embeddings must be 16-byte aligned");
  RGNN_REQUIRE(grad_h != h, "rgat_backward: grad_node_embeddings must not alias node_embeddings");
  const int V = plan->V, Vt = plan->Vt, L = plan->L, D = d_out, K = num_heads;
  RgatBwdParams ep;
  RgatAttOut att_out;
  for (int l = 0; l < L; ++l) {
    RGNN_REQUIRE(edge_weights[l] != nullptr, "rgat_backward: edge weight %d is NULL", l);
    RGNN_REQUIRE(attention[l] != nullptr && aligned16(attention[l]), "rgat_backward: attention vector %d is NULL / misaligned", l);
    RGNN_REQUIRE(grad_edge_weights == nullptr || (grad_edge_weights[l] != nullptr && aligned16(grad_edge_weights[l])),
                 "rgat_backward: grad edge weight %d is NULL / misaligned", l);
    RGNN_REQUIRE(grad_attention == nullptr || grad_attention[l] != nullptr, "rgat_backward: grad attention %d is NULL", l);
    ep.att.att[l] = attention[l];
    att_out.ptr[l] = grad_attention != nullptr ? grad_attention[l] : nullptr;
  }

  // every carve-out and the largest weight-image scratch of the two dense contractions, before anything is enqueued
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);
  float* dT = ar.floats((size_t)V * L * D);
  float* ssrc = ar.floats((size_t)V * L * K);
  float* stgt = ar.floats((size_t)V * L * K);
  float* dsrc = ar.floats((size_t)V * L * K);
  float* dtgt = ar.floats((size_t)Vt * L * K);
  float* d_o = ar.floats((size_t)Vt * D);
  float* stats = ar.floats((size_t)3 * Vt * K);
  float* att_part = grad_attention != nullptr ? ar.floats((size_t)rgat_att_blocks(V) * L * 2 * D + 4) : nullptr;
  float* tn_scratch = grad_edge_weights != nullptr ? ar.floats(gemm_tn_scratch_floats(d_in, L * D, V)) : nullptr;
  GemmParams gT, gH;
  gT.A1 = h; gT.lda1 = d_in; gT.K1 = d_in; gT.M = V; gT.N = D; gT.C = T; gT.ldc = L * D; gT.ldb1 = D;
  gT.batch_mode = BATCH_SHARED_A; gT.batch = L;
  gH.A1 = dT; gH.lda1 = L * D; gH.K1 = L * D; gH.M = V; gH.N = d_in; gH.C = grad_h; gH.ldc = d_in; gH.ldb1 = D;
  gH.batch_mode = BATCH_K_BLOCKS_T; gH.batch = L; gH.k_block = D;
  for (int l = 0; l < L; ++l) {
    gT.bptr[l] = edge_weights[l]; gH.bptr[l] = edge_weights[l];
    gT.bptr2[l] = gH.bptr2[l] = nullptr;
  }
  size_t pack = gemm_tc_pack_bytes(gT);
  if (grad_h != nullptr) pack = std::max(pack, gemm_tc_pack_bytes(gH));
  {
    const size_t mark = ar.used;
    ar.floats(pack / sizeof(float));
    RGNN_PROPAGATE(check_ws(ar, "rgat_backward"));
    ar.used = mark;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));   // T reads the halo rows

  // forward tables: T and the per-head scores (every head width)
  if (V > 0) {
    RGNN_PROPAGATE(run_gemm(gT, ar, stream));
    RGNN_PROPAGATE(launch_rgat_scores(T, V, L, D, K, ep.att, ssrc, stgt, stream));
  }
  ep.V = V; ep.Vt = Vt; ep.L = L; ep.D = D; ep.K = K; ep.act = activation;
  ep.seg_off = plan->seg_off; ep.e_src = plan->e_src; ep.e_type = plan->e_type;
  ep.heavy_list = plan->heavy_list; ep.heavy_count = plan->err_flag + 1;
  ep.rev_off = plan->rev_seg_off; ep.rev_tgt = plan->rev_src;
  ep.rev_heavy_list = plan->rev_heavy_list; ep.rev_heavy_count = plan->err_flag + 2;
  ep.T = T; ep.s_src = ssrc; ep.s_tgt = stgt; ep.grad_out = grad_out;
  ep.d_o = d_o; ep.stat_m = stats; ep.stat_den = stats + (size_t)Vt * K; ep.stat_c = stats + (size_t)2 * Vt * K;
  ep.D_tgt = dtgt; ep.D_src = dsrc; ep.dT = dT;
  RGNN_PROPAGATE(launch_rgat_edge_backward(ep, plan->num_heavy_host, stream));

  // the outputs, each written once
  if (grad_attention != nullptr) RGNN_PROPAGATE(launch_rgat_att_backward(ep, att_part, att_out, stream));
  if (grad_edge_weights != nullptr) {
    GemmTnOut tn;
    tn.block_cols = D; tn.ld = D;
    for (int l = 0; l < L; ++l) tn.ptr[l] = grad_edge_weights[l];
    RGNN_PROPAGATE(launch_gemm_tn(h, d_in, dT, L * D, d_in, L * D, V, tn, tn_scratch, stream));
  }
  if (grad_h != nullptr && V > 0) RGNN_PROPAGATE(run_gemm(gH, ar, stream));
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/gnn_film.py:8-122
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_film_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                 const float* const* edge_weights, const float* const* film_weights,
                                 const float* num_incoming, const float* ln_gamma, const float* ln_beta,
                                 int activation, int aggregation, int normalize, int num_timesteps, float* out,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "gnn_film"));
  RGNN_PROPAGATE(check_act(activation, "gnn_film"));
  RGNN_PROPAGATE(check_agg(aggregation, "gnn_film"));
  RGNN_REQUIRE(edge_weights && film_weights && ln_gamma && ln_beta, "gnn_film: NULL weight pointer");
  RGNN_REQUIRE(aligned16(ln_gamma) && aligned16(ln_beta), "gnn_film: layer-norm parameters must be 16-byte aligned");
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "gnn_film: normalize_by_num_incoming needs type_to_num_incoming_edges");
  const int V = plan->V, L = plan->L, D = d_out;
  for (int l = 0; l < L; ++l) RGNN_REQUIRE(edge_weights[l] && film_weights[l], "gnn_film: weight %d is NULL", l);
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);
  float* FW = ar.floats((size_t)V * L * 2 * D);
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * D); buf[1] = ar.floats((size_t)V * D); }
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, D);
  RGNN_PROPAGATE(check_ws(ar, "gnn_film"));

  const float* cur = h;
  int din = d_in;
  for (int t = 0; t < num_timesteps; ++t) {                                   // gnn_film.py:85
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    // [gamma | beta] = F_l h_v for the wanted target rows (:102).  This GEMM goes FIRST: it reads owned rows only, so on a
    // sharded plan it overlaps a pending halo exchange (rgnn_halo_exchange_overlapped), which transform_sources() below joins
    // before touching halo rows.
    if (plan->Vt > 0)
      RGNN_PROPAGATE(gemm_shared_a(ar, cur, plan->Vt, din, film_weights, L, 2 * D, 2 * D, FW, RGNN_ACT_LINEAR, stream));
    SegParams s;
    seg_from_plan(s, plan);
    s.D = D;
    RGNN_PROPAGATE(transform_sources(plan, ar, cur, din, D, edge_weights, T, stream, s));                        // :94 on nodes
    s.num_incoming = normalize ? num_incoming : nullptr;                      // :96-100
    s.msg_mode = MSG_FILM; s.mod_table = FW; s.mod_stride_node = (long)L * 2 * D; s.mod_stride_type = 2 * D;      // :103-108
    s.act_msg = activation;                                                   // :112 (before the sum)
    s.agg = aggregation;                                                      // :113-116
    s.ln_gamma = ln_gamma + (size_t)t * D; s.ln_beta = ln_beta + (size_t)t * D;   // :120
    s.out = dst; s.ld_out = D; s.heavy_scratch = heavy.heavy_scratch;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    cur = dst; din = D;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_gnn_film_layer: what tf.gradients produces for gnns/gnn_film.py:85-120.  No forward
// state is kept: the tables are recomputed (film_backward.cu has the math).
//   T = h . [W_0|..|W_{L-1}] (V rows), FW = h . [F_0|..|F_{L-1}] (Vt rows), a = agg act(gamma * s T + beta) (segment reduce)
//   d_a = LayerNorm backward / div                          d_ln_gamma, d_ln_beta: per-CTA partials, fixed-order sum
//   dFW[v,l] = [sum g_e s T[u,l] | sum g_e]  (CSR by target)  dT[u,l] = sum s gamma[v,l] g_e  (reverse index)
//   d_h = dT . [W_l]^T (V rows) + dFW . [F_l]^T (Vt rows)   two transposed-image GEMMs, added in that order
//   d_W_l = h^T . dT[:, l, :],  d_F_l = h[:Vt]^T . dFW[:, l, :]   TN GEMMs, split-K, deterministic
extern "C" int rgnn_film_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d_in, int32_t d_out,
                                  const float* const* edge_weights, const float* const* film_weights,
                                  const float* num_incoming, const float* ln_gamma, const float* ln_beta, int activation,
                                  int aggregation, int normalize, const float* grad_out, float* grad_h,
                                  float* const* grad_edge_weights, float* const* grad_film_weights, float* grad_ln_gamma,
                                  float* grad_ln_beta, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr && h != nullptr && grad_out != nullptr && edge_weights != nullptr && film_weights != nullptr &&
               ln_gamma != nullptr && ln_beta != nullptr, "film_backward: NULL argument");
  RGNN_REQUIRE(d_in > 0 && d_out > 0 && (d_in % 4) == 0 && (d_out % 4) == 0,
               "film_backward: dims must be positive multiples of 4 (d_in=%d, d_out=%d)", d_in, d_out);
  if (d_out > RGNN_MAX_STATE_DIM) {
    set_error("film_backward: state dim %d > %d (the layer norm holds a row per warp) is not supported", d_out, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_PROPAGATE(check_act(activation, "film_backward"));
  RGNN_PROPAGATE(check_agg(aggregation, "film_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("film_backward: the gradient of 'max' aggregation is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "film_backward: normalize_by_num_incoming needs type_to_num_incoming_edges");
  RGNN_REQUIRE(aligned16(h) && aligned16(grad_out) && aligned16(ln_gamma) && aligned16(ln_beta) && aligned16(grad_h) &&
               aligned16(grad_ln_gamma) && aligned16(grad_ln_beta), "film_backward: buffers must be 16-byte aligned");
  RGNN_REQUIRE(grad_h != h, "film_backward: grad_node_embeddings must not alias node_embeddings");
  const int V = plan->V, Vt = plan->Vt, L = plan->L, D = d_out;
  for (int l = 0; l < L; ++l) {
    RGNN_REQUIRE(edge_weights[l] != nullptr && film_weights[l] != nullptr, "film_backward: weight %d is NULL", l);
    RGNN_REQUIRE(grad_edge_weights == nullptr || (grad_edge_weights[l] != nullptr && aligned16(grad_edge_weights[l])),
                 "film_backward: grad edge weight %d is NULL / misaligned", l);
    RGNN_REQUIRE(grad_film_weights == nullptr || (grad_film_weights[l] != nullptr && aligned16(grad_film_weights[l])),
                 "film_backward: grad film weight %d is NULL / misaligned", l);
  }

  // every carve-out and the largest weight-image scratch of the four dense contractions, before anything is enqueued
  Arena ar(workspace, workspace_bytes);
  float* T = ar.floats((size_t)V * L * D);
  float* FW = ar.floats((size_t)Vt * L * 2 * D);
  float* dT = ar.floats((size_t)V * L * D);
  float* dFW = ar.floats((size_t)Vt * L * 2 * D);
  float* a = ar.floats((size_t)Vt * D);                       // the aggregate, then d_a in place
  const bool want_ln = grad_ln_gamma != nullptr || grad_ln_beta != nullptr;
  float* ln_part = ar.floats((size_t)film_ln_blocks(Vt) * 2 * D + 4);
  float* gh_tail = grad_h != nullptr ? ar.floats((size_t)Vt * d_in + 4) : nullptr;   // dFW . [F_l]^T
  float* tn_scratch = nullptr;
  if (grad_edge_weights != nullptr || grad_film_weights != nullptr) {
    const size_t a1 = gemm_tn_scratch_floats(d_in, L * D, V), a2 = gemm_tn_scratch_floats(d_in, L * 2 * D, Vt);
    tn_scratch = ar.floats(a1 > a2 ? a1 : a2);
  }
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, D);
  GemmParams gT, gF, gH1, gH2;
  gT.A1 = h; gT.lda1 = d_in; gT.K1 = d_in; gT.M = V; gT.N = D; gT.C = T; gT.ldc = L * D; gT.ldb1 = D;
  gT.batch_mode = BATCH_SHARED_A; gT.batch = L;
  gF = gT;
  gF.M = Vt; gF.N = 2 * D; gF.C = FW; gF.ldc = L * 2 * D; gF.ldb1 = 2 * D;
  gH1.A1 = dT; gH1.lda1 = L * D; gH1.K1 = L * D; gH1.M = V; gH1.N = d_in; gH1.C = grad_h; gH1.ldc = d_in; gH1.ldb1 = D;
  gH1.batch_mode = BATCH_K_BLOCKS_T; gH1.batch = L; gH1.k_block = D;
  gH2 = gH1;
  gH2.A1 = dFW; gH2.lda1 = L * 2 * D; gH2.K1 = L * 2 * D; gH2.M = Vt; gH2.C = gh_tail; gH2.ldb1 = 2 * D; gH2.k_block = 2 * D;
  for (int l = 0; l < L; ++l) {
    gT.bptr[l] = edge_weights[l]; gF.bptr[l] = film_weights[l]; gH1.bptr[l] = edge_weights[l]; gH2.bptr[l] = film_weights[l];
    gT.bptr2[l] = gF.bptr2[l] = gH1.bptr2[l] = gH2.bptr2[l] = nullptr;
  }
  size_t pack = gemm_tc_pack_bytes(gT);
  if (Vt > 0) pack = std::max(pack, gemm_tc_pack_bytes(gF));
  if (grad_h != nullptr) pack = std::max(pack, std::max(gemm_tc_pack_bytes(gH1), Vt > 0 ? gemm_tc_pack_bytes(gH2) : (size_t)0));
  {
    const size_t mark = ar.used;
    ar.floats(pack / sizeof(float));
    RGNN_PROPAGATE(check_ws(ar, "film_backward"));
    ar.used = mark;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));   // T reads the halo rows

  // forward tables and the aggregate (no layer-norm epilogue)
  if (Vt > 0) RGNN_PROPAGATE(run_gemm(gF, ar, stream));
  RGNN_PROPAGATE(run_gemm(gT, ar, stream));
  {
    SegParams s;
    seg_from_plan(s, plan);
    s.D = D; s.table = T; s.stride_idx = (long)L * D; s.stride_type = D;
    s.num_incoming = normalize ? num_incoming : nullptr;
    s.msg_mode = MSG_FILM; s.mod_table = FW; s.mod_stride_node = (long)L * 2 * D; s.mod_stride_type = 2 * D;
    s.act_msg = activation; s.agg = aggregation;
    s.out = a; s.ld_out = D; s.heavy_scratch = heavy.heavy_scratch;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
  }
  FilmLnBwdParams lp;
  lp.rows = Vt; lp.D = D; lp.agg = aggregation; lp.seg_off = plan->seg_off; lp.grad_out = grad_out; lp.ln_gamma = ln_gamma;
  lp.a = a; lp.partial = ln_part;
  RGNN_PROPAGATE(launch_film_ln_backward(lp, stream));
  FilmBwdParams ep;
  ep.V = V; ep.Vt = Vt; ep.L = L; ep.D = D; ep.act = activation;
  ep.seg_off = plan->seg_off; ep.e_src = plan->e_src; ep.e_type = plan->e_type;
  ep.heavy_list = plan->heavy_list; ep.heavy_count = plan->err_flag + 1;
  ep.rev_off = plan->rev_seg_off; ep.rev_tgt = plan->rev_src;
  ep.rev_heavy_list = plan->rev_heavy_list; ep.rev_heavy_count = plan->err_flag + 2;
  ep.T = T; ep.FW = FW; ep.d_a = a; ep.num_incoming = normalize ? num_incoming : nullptr; ep.scale_ld = V;
  ep.dT = dT; ep.dFW = dFW;
  RGNN_PROPAGATE(launch_film_edge_backward(ep, plan->num_heavy_host, stream));

  // the outputs, each written once
  if (want_ln) RGNN_PROPAGATE(launch_film_ln_param_reduce(ln_part, Vt, D, grad_ln_gamma, grad_ln_beta, stream));
  if (grad_edge_weights != nullptr) {
    GemmTnOut tn;
    tn.block_cols = D; tn.ld = D;
    for (int l = 0; l < L; ++l) tn.ptr[l] = grad_edge_weights[l];
    RGNN_PROPAGATE(launch_gemm_tn(h, d_in, dT, L * D, d_in, L * D, V, tn, tn_scratch, stream));
  }
  if (grad_film_weights != nullptr) {
    GemmTnOut tn;
    tn.block_cols = 2 * D; tn.ld = 2 * D;
    for (int l = 0; l < L; ++l) tn.ptr[l] = grad_film_weights[l];
    RGNN_PROPAGATE(launch_gemm_tn(h, d_in, dFW, L * 2 * D, d_in, L * 2 * D, Vt, tn, tn_scratch, stream));
  }
  if (grad_h != nullptr) {
    if (V > 0) RGNN_PROPAGATE(run_gemm(gH1, ar, stream));
    if (Vt > 0) {
      RGNN_PROPAGATE(run_gemm(gH2, ar, stream));
      RGNN_PROPAGATE(launch_add_rows(grad_h, gh_tail, (long)Vt * d_in, stream));
    }
  }
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/gnn_edge_mlp.py:7-122
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_edge_mlp_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                     const float* const* mlp_kernels, const int32_t* mlp_dims,
                                     int num_edge_hidden_layers, const float* num_incoming, const float* ln_gamma,
                                     const float* ln_beta, int activation, int aggregation, int normalize,
                                     int use_target, int num_timesteps, float* out, void* workspace,
                                     size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "gnn_edge_mlp"));
  RGNN_PROPAGATE(check_act(activation, "gnn_edge_mlp"));
  RGNN_PROPAGATE(check_agg(aggregation, "gnn_edge_mlp"));
  RGNN_REQUIRE(mlp_kernels && mlp_dims && ln_gamma && ln_beta, "gnn_edge_mlp: NULL weight pointer");
  RGNN_REQUIRE(num_edge_hidden_layers >= 0, "gnn_edge_mlp: num_edge_hidden_layers %d < 0", num_edge_hidden_layers);
  RGNN_REQUIRE(!normalize || num_incoming != nullptr, "gnn_edge_mlp: normalize_by_num_incoming needs type_to_num_incoming_edges");
  const int nl = num_edge_hidden_layers + 1;
  RGNN_REQUIRE(nl <= RGNN_MAX_MLP_LAYERS && mlp_dims[nl] == d_out, "gnn_edge_mlp: MLP output dim %d != state_dim %d", mlp_dims[nl <= RGNN_MAX_MLP_LAYERS ? nl : 0], d_out);
  RGNN_PROPAGATE(check_mlp_widths(mlp_dims, nl, d_in, d_out, "edge MLP", "gnn_edge_mlp"));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));
  const int V = plan->V, D = d_out;
  Arena ar(workspace, workspace_bytes);
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * D); buf[1] = ar.floats((size_t)V * D); }
  const size_t mark = ar.used;
  const float* cur = h;
  for (int t = 0; t < num_timesteps; ++t) {                                   // gnn_edge_mlp.py:84
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    ar.used = mark;                                                           // scratch of the previous timestep is dead
    MsgSource ms;
    RGNN_PROPAGATE(build_mlp_messages(plan, cur, d_in, mlp_kernels, mlp_dims, nl, use_target, RGNN_ACT_ELU, ar, stream, &ms));  // :76,:102
    RGNN_PROPAGATE(check_ws(ar, "gnn_edge_mlp"));
    SegParams s;
    seg_from_plan(s, plan);
    seg_from_source(s, ms);
    s.num_incoming = normalize ? num_incoming : nullptr;                      // :104-108
    s.act_msg = activation;                                                   // :112
    s.agg = aggregation;                                                      // :113-116
    s.ln_gamma = ln_gamma + (size_t)t * D; s.ln_beta = ln_beta + (size_t)t * D;   // :119
    s.out = dst; s.ld_out = D;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    cur = dst;
  }
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// gnns/rgin.py:7-142
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_rgin_forward(const rgnn_plan_t* plan, const float* h, int32_t d_in, int32_t d_out,
                                 const float* const* edge_mlp_kernels, const int32_t* edge_mlp_dims,
                                 int num_edge_mlp_hidden_layers, const float* const* aggr_kernels,
                                 const int32_t* aggr_dims, int num_aggr_mlp_hidden_layers, const float* ln_gamma,
                                 const float* ln_beta, int activation, int aggregation, int use_target,
                                 int num_timesteps, float* out, void* workspace, size_t workspace_bytes,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_PROPAGATE(check_common(plan, h, d_in, d_out, out, num_timesteps, "rgin"));
  RGNN_PROPAGATE(check_act(activation, "rgin"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgin"));
  RGNN_REQUIRE(ln_gamma && ln_beta, "rgin: NULL layer-norm parameters");
  const int nl_edge = num_edge_mlp_hidden_layers < 0 ? 0 : num_edge_mlp_hidden_layers + 1;
  const int nl_aggr = num_aggr_mlp_hidden_layers < 0 ? 0 : num_aggr_mlp_hidden_layers + 1;
  RGNN_REQUIRE(nl_edge == 0 || (edge_mlp_kernels && edge_mlp_dims), "rgin: NULL edge MLP table");
  RGNN_REQUIRE(nl_aggr == 0 || (aggr_kernels && aggr_dims), "rgin: NULL aggregation MLP table");
  RGNN_REQUIRE(nl_edge <= RGNN_MAX_MLP_LAYERS, "rgin: edge MLP too deep");
  RGNN_REQUIRE(nl_aggr <= RGNN_MAX_MLP_LAYERS, "rgin: aggregation MLP too deep");
  if (nl_edge > 0) RGNN_PROPAGATE(check_mlp_widths(edge_mlp_dims, nl_edge, d_in, d_out, "edge MLP", "rgin"));
  if (nl_aggr > 0) RGNN_PROPAGATE(check_mlp_widths(aggr_dims, nl_aggr, d_in, d_out, "aggregation MLP", "rgin"));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));
  const int V = plan->V, D = d_out;
  Arena ar(workspace, workspace_bytes);
  float* buf[2] = {nullptr, nullptr};
  if (num_timesteps > 1) { buf[0] = ar.floats((size_t)V * D); buf[1] = ar.floats((size_t)V * D); }
  const size_t mark = ar.used;
  const float* cur = h;
  for (int t = 0; t < num_timesteps; ++t) {                                   // rgin.py:103
    float* dst = (t == num_timesteps - 1) ? out : buf[t & 1];
    ar.used = mark;
    MsgSource ms;
    RGNN_PROPAGATE(build_mlp_messages(plan, cur, d_in, edge_mlp_kernels, edge_mlp_dims, nl_edge, use_target, activation, ar, stream, &ms));  // :95,:122
    RGNN_PROPAGATE(check_ws(ar, "rgin"));
    const int width = ms.width;
    SegParams s;
    seg_from_plan(s, plan);
    seg_from_source(s, ms);
    s.act_msg = (nl_edge > 0) ? activation : RGNN_ACT_LINEAR;                 // :128-129
    s.agg = aggregation;                                                      // :130-133
    if (nl_aggr == 0) {
      RGNN_REQUIRE(width == D, "rgin: message width %d != state_dim %d and no aggregation MLP maps it", width, D);
      s.act_out = activation;                                                 // :138
      s.ln_gamma = ln_gamma + (size_t)t * D; s.ln_beta = ln_beta + (size_t)t * D;   // :139
      s.out = dst; s.ld_out = D;
      RGNN_PROPAGATE(launch_seg_reduce(s, stream));
    } else {
      RGNN_REQUIRE(aggr_dims[0] == width && aggr_dims[nl_aggr] == D, "rgin: aggregation MLP dims [%d .. %d] do not match [%d .. %d]",
                   aggr_dims[0], aggr_dims[nl_aggr], width, D);
      float* agg = ar.floats((size_t)V * width);
      RGNN_PROPAGATE(check_ws(ar, "rgin"));
      s.out = agg; s.ld_out = width;
      RGNN_PROPAGATE(launch_seg_reduce(s, stream));
      const float* prev = agg;
      for (int j = 0; j < nl_aggr; ++j) {                                     // :136-137 (+ :138 fused into the last layer)
        RGNN_REQUIRE(aggr_kernels[j] != nullptr && (aggr_dims[j + 1] % 4) == 0, "rgin: aggregation MLP layer %d invalid", j);
        float* next = ar.floats((size_t)V * aggr_dims[j + 1]);
        RGNN_PROPAGATE(check_ws(ar, "rgin"));
        GemmParams g;
        g.A1 = prev; g.lda1 = aggr_dims[j]; g.K1 = aggr_dims[j];
        g.B1 = aggr_kernels[j]; g.ldb1 = aggr_dims[j + 1];
        g.M = plan->Vt; g.N = aggr_dims[j + 1]; g.C = next; g.ldc = aggr_dims[j + 1];   // agg holds the wanted target rows only
        g.act = activation;   // hidden layers: MLP activation (rgin.py:80); last layer: the explicit activation of :138
        RGNN_PROPAGATE(run_gemm(g, ar, stream));
        prev = next;
      }
      RGNN_PROPAGATE(launch_layer_norm(prev, plan->Vt, D, ln_gamma + (size_t)t * D, ln_beta + (size_t)t * D, dst, stream));  // :139
    }
    cur = dst;
  }
  return RGNN_OK;
}

// Backward of ONE timestep of sparse_rgin_layer with source-only messages: what tf.gradients produces for gnns/rgin.py:103-139.
// The message of edge (u -> v, l) depends on (u, l) only, so the edge MLP runs on the V node rows and nothing per edge is
// built.  No forward state is kept: every table is recomputed (rgin_backward.cu has the element-wise math).
//   Z_1 = h . [E_{0,1}|..|E_{L-1,1}] (shared-A GEMM), A_j = act(Z_j), Z_{j+1}[:, l] = A_j[:, l] . E_{l,j+1} (column blocks)
//   a = agg_{(u->v) in A_l} act(Z_{n_e}[u, l]) (segment reduce, Vt rows), U_k = Y_{k-1} . K_k, Y_k = act(U_k), Y_0 = a
//   dn = LayerNorm backward of n = Y_{n_a} (or act(a))          d_ln_gamma, d_ln_beta: per-CTA partials, fixed-order sum
//   dU_k = dY_k act'(U_k), dK_k = Y_{k-1}^T . dU_k (TN GEMM), dY_{k-1} = dU_k . K_k^T;  d_a = dY_0 / div(v), rows >= Vt zero
//   dQ[u, l] = sum_{(u->v) in A_l} d_a[v]   (reverse index)
//   dZ_{n_e} = dQ act'(P), dE_{l,j} = A_{j-1}[:, l]^T . dZ_j[:, l] (A_0 = h), dZ_{j-1}[:, l] = (dZ_j[:, l] . E_{l,j}^T) act'(Z_{j-1})
//   d_h = dZ_1 . [E_{0,1}|..|E_{L-1,1}]^T (V rows);  edge MLP None: d_h = sum_l dQ[:, l] in l order
// The per-type transposed product dZ_j[:, l] . E_{l,j}^T is one BATCH_K_BLOCKS_T launch per type (see DESIGN.md 5.4f).
extern "C" int rgnn_rgin_backward(const rgnn_plan_t* plan_c, const float* h, int32_t d_in, int32_t d_out,
                                  const float* const* edge_mlp_kernels, const int32_t* edge_mlp_dims,
                                  int num_edge_mlp_hidden_layers, const float* const* aggr_kernels, const int32_t* aggr_dims,
                                  int num_aggr_mlp_hidden_layers, const float* ln_gamma, const float* ln_beta, int activation,
                                  int aggregation, int use_target, const float* grad_out, float* grad_h,
                                  float* const* grad_edge_mlp_kernels, float* const* grad_aggr_kernels, float* grad_ln_gamma,
                                  float* grad_ln_beta, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);   // the reverse index is built lazily inside the plan
  RGNN_REQUIRE(plan != nullptr, "rgin_backward: plan is NULL");
  RGNN_REQUIRE(h != nullptr, "rgin_backward: node_embeddings is NULL");
  RGNN_REQUIRE(ln_gamma != nullptr, "rgin_backward: ln_gamma is NULL");
  RGNN_REQUIRE(ln_beta != nullptr, "rgin_backward: ln_beta is NULL");
  RGNN_REQUIRE(grad_out != nullptr, "rgin_backward: grad_out is NULL");
  RGNN_REQUIRE(d_in > 0 && d_out > 0 && (d_in % 4) == 0 && (d_out % 4) == 0,
               "rgin_backward: d_in / d_out must be positive multiples of 4 (d_in=%d, d_out=%d)", d_in, d_out);
  if (use_target) {
    set_error("rgin_backward: use_target_state_as_input = 1 (target-conditioned messages) is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  if (d_out > RGNN_MAX_STATE_DIM) {
    set_error("rgin_backward: d_out %d > %d (the layer norm holds a row per warp) is not supported", d_out, RGNN_MAX_STATE_DIM);
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_PROPAGATE(check_act(activation, "rgin_backward"));
  RGNN_PROPAGATE(check_agg(aggregation, "rgin_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("rgin_backward: the gradient of 'max' aggregation is not implemented in this build");
    return RGNN_E_UNSUPPORTED;
  }
  const int n_e = num_edge_mlp_hidden_layers < 0 ? 0 : num_edge_mlp_hidden_layers + 1;
  const int n_a = num_aggr_mlp_hidden_layers < 0 ? 0 : num_aggr_mlp_hidden_layers + 1;
  RGNN_REQUIRE(n_e <= RGNN_MAX_MLP_LAYERS, "rgin_backward: edge MLP with %d layers exceeds the supported %d", n_e, RGNN_MAX_MLP_LAYERS);
  RGNN_REQUIRE(n_a <= RGNN_MAX_MLP_LAYERS, "rgin_backward: aggregation MLP with %d layers exceeds the supported %d", n_a,
               RGNN_MAX_MLP_LAYERS);
  const int V = plan->V, Vt = plan->Vt, L = plan->L, D = d_out;
  const int32_t* ed = edge_mlp_dims;
  const int32_t* ad = aggr_dims;
  if (n_e > 0) {
    RGNN_REQUIRE(edge_mlp_kernels != nullptr, "rgin_backward: edge_mlp_kernels is NULL");
    RGNN_REQUIRE(ed != nullptr, "rgin_backward: edge_mlp_dims is NULL");
    RGNN_REQUIRE(ed[0] == d_in, "rgin_backward: edge_mlp_dims[0] = %d does not match d_in %d", ed[0], d_in);
    for (int j = 1; j <= n_e; ++j)
      RGNN_REQUIRE(ed[j] > 0 && (ed[j] % 4) == 0, "rgin_backward: edge_mlp_dims[%d] = %d must be a positive multiple of 4", j, ed[j]);
    RGNN_PROPAGATE(check_mlp_widths(ed, n_e, d_in, d_out, "edge MLP", "rgin_backward"));
    for (int i = 0; i < L * n_e; ++i) RGNN_REQUIRE(edge_mlp_kernels[i] != nullptr, "rgin_backward: edge MLP kernel %d is NULL", i);
  }
  const int width = n_e > 0 ? ed[n_e] : d_in;   // message width
  if (n_a > 0) {
    RGNN_REQUIRE(aggr_kernels != nullptr, "rgin_backward: aggr_kernels is NULL");
    RGNN_REQUIRE(ad != nullptr, "rgin_backward: aggr_dims is NULL");
    RGNN_REQUIRE(ad[0] == width && ad[n_a] == D, "rgin_backward: aggr_dims [%d .. %d] do not match [%d .. %d]", ad[0], ad[n_a], width, D);
    for (int k = 1; k <= n_a; ++k)
      RGNN_REQUIRE(ad[k] > 0 && (ad[k] % 4) == 0, "rgin_backward: aggr_dims[%d] = %d must be a positive multiple of 4", k, ad[k]);
    RGNN_PROPAGATE(check_mlp_widths(ad, n_a, d_in, d_out, "aggregation MLP", "rgin_backward"));
    for (int k = 0; k < n_a; ++k) RGNN_REQUIRE(aggr_kernels[k] != nullptr, "rgin_backward: aggregation MLP kernel %d is NULL", k);
  } else {
    RGNN_REQUIRE(width == D, "rgin_backward: message width %d != d_out %d and no aggregation MLP maps it", width, D);
  }
  RGNN_REQUIRE(aligned16(h) && aligned16(grad_out) && aligned16(ln_gamma) && aligned16(ln_beta),
               "rgin_backward: node_embeddings / grad_out / ln_gamma / ln_beta must be 16-byte aligned");
  RGNN_REQUIRE(aligned16(grad_h) && aligned16(grad_ln_gamma) && aligned16(grad_ln_beta),
               "rgin_backward: grad_node_embeddings / grad_ln_gamma / grad_ln_beta must be 16-byte aligned");
  RGNN_REQUIRE(grad_h == nullptr || (grad_h != h && grad_h != grad_out),
               "rgin_backward: grad_node_embeddings must not alias node_embeddings or grad_out");
  const bool want_e = grad_edge_mlp_kernels != nullptr && n_e > 0;
  const bool want_a = grad_aggr_kernels != nullptr && n_a > 0;
  if (want_e)
    for (int i = 0; i < L * n_e; ++i)
      RGNN_REQUIRE(grad_edge_mlp_kernels[i] != nullptr && aligned16(grad_edge_mlp_kernels[i]),
                   "rgin_backward: grad edge MLP kernel %d is NULL / misaligned", i);
  if (want_a)
    for (int k = 0; k < n_a; ++k)
      RGNN_REQUIRE(grad_aggr_kernels[k] != nullptr && aligned16(grad_aggr_kernels[k]),
                   "rgin_backward: grad aggregation MLP kernel %d is NULL / misaligned", k);

  // every carve-out and the largest weight-image scratch of the dense contractions, before anything is enqueued
  Arena ar(workspace, workspace_bytes);
  float* Z[RGNN_MAX_MLP_LAYERS + 1] = {};   // Z_j [V, L, ed[j]], then dZ_j in place
  float* Aj[RGNN_MAX_MLP_LAYERS + 1] = {};  // act(Z_j), j < n_e
  float* U[RGNN_MAX_MLP_LAYERS + 1] = {};   // U_k [Vt, ad[k]], then dU_k in place
  float* Y[RGNN_MAX_MLP_LAYERS + 1] = {};   // Y_k = act(U_k) [Vt, ad[k]], then dY_k; Y_0 = a
  int gw = width;                           // dQ, then each dA_{j-1}: [V, L, <= gw]
  for (int j = 1; j <= n_e; ++j) Z[j] = ar.floats((size_t)V * L * ed[j]);
  for (int j = 1; j < n_e; ++j) { Aj[j] = ar.floats((size_t)V * L * ed[j]); gw = std::max(gw, (int)ed[j]); }
  float* G = ar.floats((size_t)V * L * gw);
  float* a = ar.floats((size_t)V * width);   // the aggregate, then d_a (every row: the reverse gather reads any target)
  Y[0] = a;
  for (int k = 1; k <= n_a; ++k) U[k] = ar.floats((size_t)Vt * ad[k]);
  for (int k = 1; k < n_a; ++k) Y[k] = ar.floats((size_t)Vt * ad[k]);
  float* nrm = ar.floats((size_t)Vt * D);   // n, then dn in place
  if (n_a > 0) Y[n_a] = nrm;
  float* ln_part = ar.floats((size_t)film_ln_blocks(Vt) * 2 * D + 4);
  float* tn_scratch = nullptr;
  {
    size_t n = 0;
    if (want_e) {
      n = gemm_tn_scratch_floats(d_in, L * ed[1], V);
      for (int j = 2; j <= n_e; ++j) n = std::max(n, gemm_tn_scratch_floats(ed[j - 1], ed[j], V));
    }
    if (want_a)
      for (int k = 1; k <= n_a; ++k) n = std::max(n, gemm_tn_scratch_floats(ad[k - 1], ad[k], Vt));
    if (n > 0) tn_scratch = ar.floats(n);
  }
  SegParams heavy;
  seg_heavy_scratch(heavy, plan, ar, width);

  // the dense contractions
  const float* bp[RGNN_MAX_EDGE_TYPES];
  auto fwd_edge = [&](int j) {   // Z_j = A_{j-1} . E_{l,j} per type (j = 1: the shared-A GEMM on h)
    GemmParams g;
    g.M = V; g.N = ed[j]; g.C = Z[j]; g.ldc = L * ed[j]; g.ldb1 = ed[j]; g.batch = L;
    if (j == 1) { g.A1 = h; g.lda1 = d_in; g.K1 = d_in; g.batch_mode = BATCH_SHARED_A; }
    else { g.A1 = Aj[j - 1]; g.lda1 = L * ed[j - 1]; g.K1 = ed[j - 1]; g.batch_mode = BATCH_COL_BLOCKS; }
    for (int l = 0; l < L; ++l) { g.bptr[l] = edge_mlp_kernels[l * n_e + j - 1]; g.bptr2[l] = nullptr; }
    return g;
  };
  auto bwd_edge = [&](int j, int l) {   // dA_{j-1}[:, l] = dZ_j[:, l] . E_{l,j}^T  (j >= 2)
    GemmParams g;
    g.A1 = Z[j] + (size_t)l * ed[j]; g.lda1 = L * ed[j]; g.K1 = ed[j]; g.M = V; g.N = ed[j - 1];
    g.C = G + (size_t)l * ed[j - 1]; g.ldc = L * ed[j - 1]; g.ldb1 = ed[j];
    g.batch_mode = BATCH_K_BLOCKS_T; g.batch = 1; g.k_block = ed[j]; g.bptr[0] = edge_mlp_kernels[l * n_e + j - 1]; g.bptr2[0] = nullptr;
    return g;
  };
  auto fwd_aggr = [&](int k) {   // U_k = Y_{k-1} . K_k
    GemmParams g;
    g.A1 = Y[k - 1]; g.lda1 = ad[k - 1]; g.K1 = ad[k - 1]; g.B1 = aggr_kernels[k - 1]; g.ldb1 = ad[k];
    g.M = Vt; g.N = ad[k]; g.C = U[k]; g.ldc = ad[k];
    return g;
  };
  auto bwd_aggr = [&](int k) {   // dY_{k-1} = dU_k . K_k^T
    GemmParams g;
    g.A1 = U[k]; g.lda1 = ad[k]; g.K1 = ad[k]; g.M = Vt; g.N = ad[k - 1]; g.C = Y[k - 1]; g.ldc = ad[k - 1]; g.ldb1 = ad[k];
    g.batch_mode = BATCH_K_BLOCKS_T; g.batch = 1; g.k_block = ad[k]; g.bptr[0] = aggr_kernels[k - 1]; g.bptr2[0] = nullptr;
    return g;
  };
  GemmParams gH;   // d_h = dZ_1 . [E_{0,1}|..|E_{L-1,1}]^T
  if (n_e > 0) {
    gH.A1 = Z[1]; gH.lda1 = L * ed[1]; gH.K1 = L * ed[1]; gH.M = V; gH.N = d_in; gH.C = grad_h; gH.ldc = d_in; gH.ldb1 = ed[1];
    gH.batch_mode = BATCH_K_BLOCKS_T; gH.batch = L; gH.k_block = ed[1];
    for (int l = 0; l < L; ++l) { gH.bptr[l] = edge_mlp_kernels[l * n_e]; gH.bptr2[l] = nullptr; }
  }
  size_t pack = 0;
  if (V > 0) {
    for (int j = 1; j <= n_e; ++j) pack = std::max(pack, gemm_tc_pack_bytes(fwd_edge(j)));
    for (int j = 2; j <= n_e; ++j)
      for (int l = 0; l < L; ++l) pack = std::max(pack, gemm_tc_pack_bytes(bwd_edge(j, l)));
    if (grad_h != nullptr && n_e > 0) pack = std::max(pack, gemm_tc_pack_bytes(gH));
  }
  if (Vt > 0)
    for (int k = 1; k <= n_a; ++k) pack = std::max(pack, std::max(gemm_tc_pack_bytes(fwd_aggr(k)), gemm_tc_pack_bytes(bwd_aggr(k))));
  {
    const size_t mark = ar.used;
    ar.floats(pack / sizeof(float));
    RGNN_PROPAGATE(check_ws(ar, "rgin_backward"));
    ar.used = mark;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  RGNN_PROPAGATE(plan_wait_sources(plan, stream));   // the edge MLP reads the halo rows

  // forward: the edge MLP on the node rows, the aggregate, the aggregation MLP
  for (int j = 1; j <= n_e; ++j) {
    if (V > 0) RGNN_PROPAGATE(run_gemm(fwd_edge(j), ar, stream));
    if (j < n_e) RGNN_PROPAGATE(launch_rgin_act(Z[j], (long)V * L * ed[j], activation, Aj[j], stream));
  }
  {
    SegParams s;
    seg_from_plan(s, plan);
    s.D = width;
    if (n_e > 0) { s.table = Z[n_e]; s.stride_idx = (long)L * width; s.stride_type = width; s.act_msg = activation; }   // :128-129
    else { s.table = h; s.stride_idx = d_in; s.stride_type = 0; }
    s.agg = aggregation; s.out = a; s.ld_out = width; s.heavy_scratch = heavy.heavy_scratch;
    RGNN_PROPAGATE(launch_seg_reduce(s, stream));
  }
  for (int k = 1; k <= n_a; ++k) {
    if (Vt > 0) RGNN_PROPAGATE(run_gemm(fwd_aggr(k), ar, stream));
    RGNN_PROPAGATE(launch_rgin_act(U[k], (long)Vt * ad[k], activation, Y[k], stream));
  }
  if (n_a == 0) RGNN_PROPAGATE(launch_rgin_act(a, (long)Vt * D, activation, nrm, stream));   // :138

  // layer norm, then the aggregation MLP down to d_a
  FilmLnBwdParams lp;
  lp.rows = Vt; lp.D = D; lp.agg = RGNN_AGG_SUM; lp.seg_off = plan->seg_off; lp.grad_out = grad_out; lp.ln_gamma = ln_gamma;
  lp.a = nrm; lp.partial = ln_part;
  RGNN_PROPAGATE(launch_film_ln_backward(lp, stream));
  RginGradParams gp;
  gp.act = activation;
  if (n_a == 0) {
    gp.rows = V; gp.valid = Vt; gp.width = width; gp.agg = aggregation; gp.seg_off = plan->seg_off;
    gp.g = nrm; gp.x = a; gp.out = a;
    RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
  } else {
    gp.rows = gp.valid = Vt; gp.width = D; gp.g = nrm; gp.x = U[n_a]; gp.out = U[n_a];
    RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
    for (int k = n_a; k >= 1; --k) {
      if (want_a) {
        GemmTnOut tn;
        tn.block_cols = ad[k]; tn.ld = ad[k]; tn.ptr[0] = grad_aggr_kernels[k - 1];
        RGNN_PROPAGATE(launch_gemm_tn(Y[k - 1], ad[k - 1], U[k], ad[k], ad[k - 1], ad[k], Vt, tn, tn_scratch, stream));
      }
      if (Vt > 0) RGNN_PROPAGATE(run_gemm(bwd_aggr(k), ar, stream));   // dY_{k-1} overwrites Y_{k-1} after d_K_k read it
      if (k > 1) {
        gp.rows = gp.valid = Vt; gp.width = ad[k - 1]; gp.g = Y[k - 1]; gp.x = U[k - 1]; gp.out = U[k - 1];
        RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
      }
    }
    gp.rows = V; gp.valid = Vt; gp.width = width; gp.act = RGNN_ACT_LINEAR; gp.agg = aggregation; gp.seg_off = plan->seg_off;
    gp.g = a; gp.x = nullptr; gp.out = a;
    RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
  }

  // the source side: dQ[u, l] = sum over the edges (u -> v) of type l of d_a[v]; every (u, l) row is written
  {
    SegParams r;   // reverse index: segment = (source u, type l); gathered row = d_a[original target]
    r.V = V * L; r.L = L; r.D = width;
    r.seg_off = plan->rev_seg_off; r.e_idx = plan->rev_src; r.e_type = plan->rev_type;
    r.table = a; r.stride_idx = width; r.stride_type = 0;
    r.heavy_list = plan->rev_heavy_list; r.heavy_count = plan->err_flag + 2;
    r.heavy_threshold = RGNN_HEAVY_SEGMENT; r.heavy_known = -1;
    r.agg = RGNN_AGG_SUM; r.out = G; r.ld_out = width;
    RGNN_PROPAGATE(launch_seg_reduce(r, stream));
  }

  // the edge MLP, from the message down to h
  if (n_e == 0) {
    if (grad_h != nullptr) RGNN_PROPAGATE(launch_rgin_type_sum(G, V, L, d_in, grad_h, stream));
  } else {
    gp = RginGradParams();
    gp.act = activation; gp.rows = gp.valid = V; gp.width = L * width; gp.g = G; gp.x = Z[n_e]; gp.out = Z[n_e];
    RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
    for (int j = n_e; j >= 2; --j) {
      if (want_e)
        for (int l = 0; l < L; ++l) {
          GemmTnOut tn;
          tn.block_cols = ed[j]; tn.ld = ed[j]; tn.ptr[0] = grad_edge_mlp_kernels[l * n_e + j - 1];
          RGNN_PROPAGATE(launch_gemm_tn(Aj[j - 1] + (size_t)l * ed[j - 1], L * ed[j - 1], Z[j] + (size_t)l * ed[j], L * ed[j],
                                        ed[j - 1], ed[j], V, tn, tn_scratch, stream));
        }
      if (V > 0)
        for (int l = 0; l < L; ++l) RGNN_PROPAGATE(run_gemm(bwd_edge(j, l), ar, stream));
      gp.width = L * ed[j - 1]; gp.g = G; gp.x = Z[j - 1]; gp.out = Z[j - 1];
      RGNN_PROPAGATE(launch_rgin_act_grad(gp, stream));
    }
    if (want_e) {
      GemmTnOut tn;
      tn.block_cols = ed[1]; tn.ld = ed[1];
      for (int l = 0; l < L; ++l) tn.ptr[l] = grad_edge_mlp_kernels[l * n_e];
      RGNN_PROPAGATE(launch_gemm_tn(h, d_in, Z[1], L * ed[1], d_in, L * ed[1], V, tn, tn_scratch, stream));
    }
    if (grad_h != nullptr && V > 0) RGNN_PROPAGATE(run_gemm(gH, ar, stream));
  }
  if (grad_ln_gamma != nullptr || grad_ln_beta != nullptr)
    RGNN_PROPAGATE(launch_film_ln_param_reduce(ln_part, Vt, D, grad_ln_gamma, grad_ln_beta, stream));
  return RGNN_OK;
}

// ---------------------------------------------------------------------------------------------
// building blocks
// ---------------------------------------------------------------------------------------------
extern "C" int rgnn_segment_aggregate(const rgnn_plan_t* plan, const float* data, int32_t d, int aggregation,
                                      float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(plan != nullptr && data != nullptr && out != nullptr, "segment_aggregate: NULL argument");
  RGNN_PROPAGATE(check_agg(aggregation, "segment_aggregate"));
  SegParams s;
  seg_from_plan(s, plan);
  s.e_idx = plan->e_orig; s.table = data; s.stride_idx = d; s.stride_type = 0; s.D = d;
  s.agg = aggregation; s.out = out; s.ld_out = d;
  return launch_seg_reduce(s, stream);
}

// The edge stage on per-node transformed states (rgcn.py:84-112, ggnn.py:76-90 after re-association):
// out[v] = agg_{l, (u,v) in A_l} s_{l,v} * table[u, l, :]
extern "C" int rgnn_edge_aggregate_forward(const rgnn_plan_t* plan, const float* table, int32_t d, const float* num_incoming,
                                           int aggregation, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(plan != nullptr && table != nullptr && out != nullptr, "edge_aggregate: NULL argument");
  RGNN_REQUIRE(d > 0 && (d % 4) == 0 && aligned16(table) && aligned16(out), "edge_aggregate: d must be a positive multiple of 4, rows 16-byte aligned");
  RGNN_PROPAGATE(check_agg(aggregation, "edge_aggregate"));
  SegParams s;
  seg_from_plan(s, plan);
  s.D = d; s.table = table; s.stride_idx = (long)plan->L * d; s.stride_type = d;
  s.num_incoming = num_incoming;
  s.agg = aggregation; s.out = out; s.ld_out = d;
  return launch_seg_reduce(s, stream);
}

// d_table[u, l, :] = sum_{(u,v) in A_l} s_{l,v} * grad_out[v, :] / div(v)   (reverse index: segments = (source, type))
extern "C" int rgnn_edge_aggregate_backward(const rgnn_plan_t* plan_c, const float* grad_out, int32_t d,
                                            const float* num_incoming, int aggregation, float* d_table, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  rgnn_plan* plan = const_cast<rgnn_plan*>(plan_c);
  RGNN_REQUIRE(plan != nullptr && grad_out != nullptr && d_table != nullptr, "edge_aggregate_backward: NULL argument");
  RGNN_REQUIRE(d > 0 && (d % 4) == 0 && aligned16(grad_out) && aligned16(d_table), "edge_aggregate_backward: d must be a positive multiple of 4, rows 16-byte aligned");
  RGNN_PROPAGATE(check_agg(aggregation, "edge_aggregate_backward"));
  if (aggregation == RGNN_AGG_MAX) {
    set_error("edge_aggregate_backward: the gradient of 'max' aggregation is not implemented in this kernel");
    return RGNN_E_UNSUPPORTED;
  }
  RGNN_PROPAGATE(plan_ensure_reverse(plan, stream));
  const int V = plan->V, L = plan->L;
  const float* d_agg = grad_out;
  float* scratch = nullptr;
  if (aggregation != RGNN_AGG_SUM) {   // mean / sqrt_n: divide by the segment size first
    RGNN_CHECK_CUDA(cudaMallocAsync(&scratch, sizeof(float) * (size_t)(V > 0 ? V : 1) * d, stream));
    const int rc = launch_act_backward(grad_out, grad_out, nullptr, V, d, RGNN_ACT_LINEAR, aggregation, plan->seg_off, scratch, stream);
    if (rc != RGNN_OK) { cudaFreeAsync(scratch, stream); return rc; }
    d_agg = scratch;
  }
  SegParams r;
  r.V = V * L; r.L = L; r.D = d;
  r.seg_off = plan->rev_seg_off; r.e_idx = plan->rev_src; r.e_type = plan->rev_type;
  r.table = d_agg; r.stride_idx = d; r.stride_type = 0;
  r.num_incoming = num_incoming; r.scale_ld = V; r.scale_by_idx = 1;
  r.heavy_list = plan->rev_heavy_list; r.heavy_count = plan->err_flag + 2;
  r.heavy_threshold = RGNN_HEAVY_SEGMENT; r.heavy_known = -1;
  r.agg = RGNN_AGG_SUM; r.out = d_table; r.ld_out = d;
  const int rc = launch_seg_reduce(r, stream);
  if (scratch != nullptr) cudaFreeAsync(scratch, stream);
  return rc;
}

// Scratch of rgnn_dense_forward / rgnn_dense_backward: the weight images of the contraction(s) + the split-K partial tiles.
extern "C" size_t rgnn_dense_workspace_bytes(int32_t m, int32_t k, int32_t n) {
  if (m < 0 || k <= 0 || n <= 0) return 0;
  GemmParams f;
  f.M = m; f.N = n; f.K1 = k; f.lda1 = k; f.ldb1 = n; f.ldc = n;
  GemmParams t;
  t.M = m; t.N = k; t.K1 = n; t.lda1 = n; t.ldb1 = n; t.ldc = k; t.batch_mode = BATCH_K_BLOCKS_T; t.batch = 1; t.k_block = n;
  const size_t pack = gemm_tc_pack_bytes_uncached(f) > gemm_tc_pack_bytes_uncached(t) ? gemm_tc_pack_bytes_uncached(f) : gemm_tc_pack_bytes_uncached(t);
  return align_up(pack, 256) + align_up(gemm_tn_scratch_floats(k, n, m) * sizeof(float), 256) + 512;
}

extern "C" int rgnn_dense_forward(const float* a, int32_t m, int32_t k, const float* b, int32_t n, const float* bias,
                                  int activation, float* c, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE(a && b && c, "dense: NULL argument");
  RGNN_PROPAGATE(check_act(activation, "dense"));
  GemmParams g;
  g.A1 = a; g.lda1 = k; g.K1 = k; g.B1 = b; g.ldb1 = n; g.M = m; g.N = n; g.C = c; g.ldc = n;
  g.bias = bias; g.act = activation;
  Arena ar(workspace, workspace_bytes);
  return run_gemm(g, ar, stream);
}

// gradients of the linear map C = A . B of rgnn_dense_forward (TF autodiff of tf.keras Dense, sparse_graph_model.py:253)
extern "C" int rgnn_dense_backward(const float* a, int32_t m, int32_t k, const float* b, int32_t n, const float* grad_c,
                                   float* grad_a, float* grad_b, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RGNN_REQUIRE((grad_c != nullptr || m == 0) && m >= 0 && k > 0 && n > 0 && (k % 4) == 0 && (n % 4) == 0, "dense_backward: bad arguments (m=%d k=%d n=%d)", m, k, n);
  RGNN_REQUIRE(grad_a == nullptr || m == 0 || b != nullptr, "dense_backward: grad_a needs b");
  RGNN_REQUIRE(grad_b == nullptr || a != nullptr || m == 0, "dense_backward: grad_b needs a");
  GemmParams g;
  g.A1 = grad_c; g.lda1 = n; g.K1 = n; g.M = m; g.N = k; g.C = grad_a; g.ldc = k; g.ldb1 = n;
  g.batch_mode = BATCH_K_BLOCKS_T; g.batch = 1; g.k_block = n; g.bptr[0] = b; g.bptr2[0] = nullptr;
  {   // size both contractions before launching either: a refused call must not have written grad_a already
    Arena probe(workspace, workspace_bytes);
    if (grad_a != nullptr && m > 0) { probe.floats(gemm_tc_pack_bytes(g) / sizeof(float)); if (!probe.overflow) probe.used = 0; }
    if (grad_b != nullptr) probe.floats(gemm_tn_scratch_floats(k, n, m));
    RGNN_PROPAGATE(check_ws(probe, "dense_backward"));
  }
  Arena ar(workspace, workspace_bytes);
  if (grad_a != nullptr && m > 0)     // dA = dC . B^T
    RGNN_PROPAGATE(run_gemm(g, ar, stream));
  if (grad_b != nullptr) {            // dB = A^T . dC
    GemmTnOut tn;
    tn.block_cols = n; tn.ld = n; tn.ptr[0] = grad_b;
    float* ws = ar.floats(gemm_tn_scratch_floats(k, n, m));
    RGNN_PROPAGATE(check_ws(ar, "dense_backward"));
    RGNN_PROPAGATE(launch_gemm_tn(a, k, grad_c, n, k, n, m, tn, ws, stream));
  }
  return RGNN_OK;
}

extern "C" int rgnn_layer_norm(const float* x, int32_t rows, int32_t d, const float* gamma, const float* beta,
                               float* out, void* stream_) {
  RGNN_REQUIRE(x && gamma && beta && out, "layer_norm: NULL argument");
  return launch_layer_norm(x, rows, d, gamma, beta, out, static_cast<cudaStream_t>(stream_));
}
