// seg.cuh -- edge-stage kernels: gather message rows by source, modulate, segment-reduce to the target.
#pragma once
#include "common.cuh"
#include "plan.cuh"

namespace rgnn {

enum MsgMode {
  MSG_LINEAR = 0,   // m = s * t                      (RGCN / GGNN / RGIN / materialised per-edge MLP outputs)
  MSG_FILM = 1,     // m = gamma * (s * t) + beta     (gnn_film.py:96-108)
  MSG_ADDTGT = 2,   // m = s * (t + q)                ([h_u | h_v] . W  ==  h_u.W_src + h_v.W_tgt : rgcn.py:91-96, gnn_edge_mlp.py:95-102)
};

struct SegParams {
  int V = 0, L = 1, D = 0;
  const int32_t* seg_off = nullptr;
  const int32_t* e_idx = nullptr;      // plan->e_src (tables indexed by node) or plan->e_orig (per-edge matrices)
  const int32_t* e_type = nullptr;
  const float* table = nullptr;        // message row of edge e = table + e_idx[e]*stride_idx + e_type[e]*stride_type
  long stride_idx = 0, stride_type = 0;
  const float* num_incoming = nullptr; // [L, scale_ld] fp32 -> s = 1/(c + 1e-7) (rgcn.py:100-104); NULL -> s = 1
  int scale_ld = 0;                    // row length of num_incoming (number of graph nodes)
  int scale_by_idx = 0;                // 0: c[type, v] of the segment's target v; 1: c[type, e_idx] (backward: the edge's original target)
  int msg_mode = MSG_LINEAR;
  const float* mod_table = nullptr;    // FILM: gamma at +0, beta at +D ; ADDTGT: q.  row = mod_table + v*mod_stride_node + type*mod_stride_type
  long mod_stride_node = 0, mod_stride_type = 0;
  int act_msg = RGNN_ACT_LINEAR;       // activation applied per message before the reduction
  int agg = RGNN_AGG_SUM;
  int act_out = RGNN_ACT_LINEAR;       // activation applied to the aggregate
  const float* ln_gamma = nullptr;     // non-NULL -> tf.contrib.layers.layer_norm epilogue (eps 1e-12)
  const float* ln_beta = nullptr;
  float* out = nullptr;
  int ld_out = 0;
  // degree-skew handling: targets with more than heavy_threshold incoming edges are skipped by the warp-per-target
  // kernel and reduced by a whole CTA each (seg_reduce_heavy_kernel).  heavy_list / heavy_count live in the plan.
  const int32_t* heavy_list = nullptr;
  const int* heavy_count = nullptr;    // device counter
  int heavy_threshold = 0;             // 0 = no splitting
  int heavy_known = -1;                // host copy of *heavy_count, or -1 when it was never read back
  // multi-CTA split (forward plans; needs scratch): every RGNN_HEAVY_CHUNK edges of a heavy target are one work item reduced
  // by one CTA into heavy_scratch[item, :]; a second kernel adds a target's partial rows in a fixed order and finishes the row
  const int32_t* heavy_base = nullptr; // [heavy targets] first item of heavy target i
  const int32_t* heavy_items = nullptr;// (target, chunk) pairs
  const int* heavy_item_count = nullptr;
  int heavy_items_known = -1, heavy_items_cap = 0, heavy_chunk = 0;
  float* heavy_scratch = nullptr;      // [heavy_items_cap, D] floats; NULL -> one CTA per heavy target (no split)
};
int launch_seg_reduce(const SegParams& p, cudaStream_t stream);

struct AttnTable { const float* att[RGNN_MAX_EDGE_TYPES]; };
struct RgatParams {
  int V = 0, L = 1, D = 0, K = 1;
  AttnTable att;                       // per-type attention vectors [2D] (fused-score path: s_src / s_tgt are NULL)
  const int32_t* seg_off = nullptr;
  const int32_t* e_src = nullptr;
  const int32_t* e_type = nullptr;
  const float* table = nullptr;        // T [V, L, D]
  const float* s_src = nullptr;        // [V, L, K]
  const float* s_tgt = nullptr;        // [V, L, K]
  int act_out = RGNN_ACT_LINEAR;
  float* out = nullptr;
};
int launch_seg_rgat(const RgatParams& p, cudaStream_t stream);

// gnns/rgdcn.py:121-171: messages h_u[c,:] . W[v,l,c] with a per-(target, type, channel) K x K kernel computed from the
// target's state.  wdyn [V, L, C, K, K] row-major (C = D / K).
struct RgdcnParams {
  int V = 0, L = 1, D = 0, K = 0;
  const int32_t* seg_off = nullptr;
  const int32_t* e_src = nullptr;
  const int32_t* e_type = nullptr;
  const float* h = nullptr;            // [V, D]
  const float* wdyn = nullptr;         // [V, L, D * K]
  const float* num_incoming = nullptr; // [L, scale_ld] or NULL
  int scale_ld = 0;                    // row length of num_incoming (all graph nodes; V may be fewer wanted targets)
  int agg = RGNN_AGG_SUM;
  int act_out = RGNN_ACT_LINEAR;
  float* out = nullptr;                // [V, D]
};
int launch_rgdcn_edges(const RgdcnParams& p, cudaStream_t stream);

// s_src[n,l,k] = <att_l[k*2d : k*2d+d], T[n,l,k*d:(k+1)*d]>, s_tgt with att_l[k*2d+d : (k+1)*2d]  (rgat.py:106-115)
int launch_rgat_scores(const float* table, int V, int L, int D, int K, const AttnTable& att, float* s_src,
                       float* s_tgt, cudaStream_t stream);

// X[i, :] (i in type-major original order) = act(P[src_i, type, :] + Q[tgt_i, type, :])   (pq != NULL), or
// X[i, :] = [h[src_i] | h[tgt_i]]                                                         (concat mode)
struct EdgeBuildParams {
  int L = 1, D = 0;                     // D = width of P / Q rows (or of h in concat mode)
  const int32_t* o_src = nullptr;
  const int32_t* o_tgt = nullptr;
  int32_t type_off[RGNN_MAX_EDGE_TYPES + 1];
  int max_type_edges = 0;
  const float* p = nullptr; long p_stride_node = 0, p_stride_type = 0;
  const float* q = nullptr; long q_stride_node = 0, q_stride_type = 0;   // NULL -> concat mode
  int concat = 0;
  int act = RGNN_ACT_LINEAR;
  float* x = nullptr; int ldx = 0;
};
int launch_edge_build(const EdgeBuildParams& p, cudaStream_t stream);

int launch_layer_norm(const float* x, int rows, int D, const float* gamma, const float* beta, float* out,
                      cudaStream_t stream);

// d_agg[v, :] = grad_out[v, :] * act'(.) / div(v)   -- the elementwise head of every layer backward.
// act' is evaluated from the forward OUTPUT for linear/tanh/relu/leaky_relu/elu/selu and from the
// pre-activation `pre` (must be non-NULL) for gelu.  div: 1 (sum/max), n (mean), sqrt(n) (sqrt_n), n = max(in-degree, 1).
int launch_act_backward(const float* grad_out, const float* out, const float* pre, int V, int D, int act, int agg,
                        const int32_t* seg_off, float* d_agg, cudaStream_t stream);

// ---- rgnn_film_backward (film_backward.cu) ----
// LayerNorm backward of one FiLM timestep: a [rows, D] (the recomputed aggregate) is overwritten with
// d_a = rstd (g - mean(g) - x_hat mean(g x_hat)) / div(v), g = grad_out * ln_gamma; per-CTA partial sums of grad_out * x_hat
// and grad_out go to partial [film_ln_blocks(rows), 2D] and are added in CTA order into d_gamma / d_beta (either may be NULL).
struct FilmLnBwdParams {
  int rows = 0, D = 0, agg = RGNN_AGG_SUM;
  const int32_t* seg_off = nullptr;    // divisor of mean / sqrt_n: all incoming edges of v
  const float* grad_out = nullptr;
  const float* ln_gamma = nullptr;
  float* a = nullptr;
  float* partial = nullptr;
};
constexpr int FILM_LN_MAX_BLOCKS = 2 * RGNN_WAVE_SMS;
inline int film_ln_blocks(int rows) {
  const int b = (rows + 7) / 8;
  return b < FILM_LN_MAX_BLOCKS ? b : FILM_LN_MAX_BLOCKS;
}
int launch_film_ln_backward(const FilmLnBwdParams& p, cudaStream_t stream);
int launch_film_ln_param_reduce(const float* partial, int rows, int D, float* d_gamma, float* d_beta, cudaStream_t stream);

// The two edge kernels: dFW [Vt, L, 2D] over the CSR by target, dT [V, L, D] over the reverse index.
struct FilmBwdParams {
  int V = 0, Vt = 0, L = 1, D = 0, act = RGNN_ACT_LINEAR;
  const int32_t* seg_off = nullptr; const int32_t* e_src = nullptr; const int32_t* e_type = nullptr;
  const int32_t* heavy_list = nullptr; const int* heavy_count = nullptr;          // targets above RGNN_HEAVY_SEGMENT
  const int32_t* rev_off = nullptr; const int32_t* rev_tgt = nullptr;             // segment u * L + l, entry = target
  const int32_t* rev_heavy_list = nullptr; const int* rev_heavy_count = nullptr;
  const float* T = nullptr;            // [V, L, D]   h . [W_0 | .. | W_{L-1}]
  const float* FW = nullptr;           // [Vt, L, 2D] h . [F_0 | .. | F_{L-1}]  (gamma | beta)
  const float* d_a = nullptr;          // [Vt, D]
  const float* num_incoming = nullptr; // [L, scale_ld] or NULL
  int scale_ld = 0;
  float* dT = nullptr;
  float* dFW = nullptr;
};
int launch_film_edge_backward(const FilmBwdParams& p, int heavy_known, cudaStream_t stream);
// y[0:n] += x[0:n]  (n % 4 == 0)
int launch_add_rows(float* y, const float* x, long n, cudaStream_t stream);

// ---- rgnn_rgat_backward (rgat_backward.cu) ----
// The edge kernels: d_o [Vt, D], the softmax statistics m / den / c [Vt, K] and D_tgt [Vt, L, K] over the CSR by target;
// dT [V, L, D] and D_src [V, L, K] over the reverse index.
struct RgatBwdParams {
  int V = 0, Vt = 0, L = 1, D = 0, K = 1, act = RGNN_ACT_LINEAR;
  AttnTable att;                       // per-type attention vectors [2D]
  const int32_t* seg_off = nullptr; const int32_t* e_src = nullptr; const int32_t* e_type = nullptr;
  const int32_t* heavy_list = nullptr; const int* heavy_count = nullptr;          // targets above RGNN_HEAVY_SEGMENT
  const int32_t* rev_off = nullptr; const int32_t* rev_tgt = nullptr;             // segment u * L + l, entry = target
  const int32_t* rev_heavy_list = nullptr; const int* rev_heavy_count = nullptr;
  const float* T = nullptr;            // [V, L, D]   h . [W_0 | .. | W_{L-1}]
  const float* s_src = nullptr;        // [V, L, K]
  const float* s_tgt = nullptr;        // [V, L, K]
  const float* grad_out = nullptr;     // [Vt, D]
  float* d_o = nullptr;                // [Vt, D]    act'(o) * grad_out
  float* stat_m = nullptr;             // [Vt, K]    softmax max
  float* stat_den = nullptr;           // [Vt, K]    softmax denominator
  float* stat_c = nullptr;             // [Vt, K]    <d_o, o> per head
  float* D_tgt = nullptr;              // [Vt, L, K] sum of d_x over the (target, type) run
  float* D_src = nullptr;              // [V, L, K]  sum of d_x over the (source, type) segment
  float* dT = nullptr;                 // [V, L, D]
};
int launch_rgat_edge_backward(const RgatBwdParams& p, int heavy_known, cudaStream_t stream);
// d_att_l [2D] from T, D_src and D_tgt: per-CTA partial sums in partial [rgat_att_blocks(V), L, 2D], added in CTA order
struct RgatAttOut { float* ptr[RGNN_MAX_EDGE_TYPES]; };
constexpr int RGAT_ATT_MAX_BLOCKS = 2 * RGNN_WAVE_SMS;
inline int rgat_att_blocks(int V) {
  const int b = (V + 63) / 64;
  return b < RGAT_ATT_MAX_BLOCKS ? b : RGAT_ATT_MAX_BLOCKS;
}
int launch_rgat_att_backward(const RgatBwdParams& p, float* partial, const RgatAttOut& out, cudaStream_t stream);

// ---- rgnn_ggnn_backward (ggnn_backward.cu) ----
// The element-wise parts of the cell backward over the wanted target rows [0, rows).  GRU: a / da [rows, 3D] hold
// [a_z | a_r | a_h] / [da_z | da_r | da_h]; stage 0 writes da_z, da_h and e = g z, stage 1 (after d(rh) = da_h . R_h^T) writes
// da_r and adds d(rh) r to e.  RNN: a / da [rows, D] (da may be a).  e may be NULL (no d_h wanted).
struct GgnnCellBwdParams {
  int rows = 0, D = 0, act = RGNN_ACT_LINEAR;
  const float* grad_out = nullptr;     // [rows, D]
  const float* h = nullptr;            // [rows, D]  this timestep's input
  const float* a = nullptr;            // pre-activations
  float* da = nullptr;
  const float* drh = nullptr;          // [rows, D]  GRU stage 1
  float* e = nullptr;                  // [rows, D]  element-wise terms of the cell's d_h
};
int launch_ggnn_cell_backward(const GgnnCellBwdParams& p, int cell_kind, int stage, cudaStream_t stream);
// rh [rows, D] = hs(a_r) * h, a [rows, 3D]
int launch_ggnn_gru_rh(const float* a, const float* h, int rows, int D, float* rh, cudaStream_t stream);
// dm [V, D]: rows < Vt divided by the mean / sqrt_n divisor, rows >= Vt zeroed
int launch_ggnn_dm_finish(float* dm, int V, int Vt, int D, int agg, const int32_t* seg_off, cudaStream_t stream);
// y[0:n] += e[0:n] + f[0:n] (f may be NULL)
int launch_ggnn_add_cell_grad(float* y, const float* e, const float* f, long n, cudaStream_t stream);
// out [N] = column sums of x [rows, N]: per-CTA partial sums in partial [ggnn_colsum_blocks(rows), N], added in CTA order
constexpr int GGNN_COLSUM_MAX_BLOCKS = 2 * RGNN_WAVE_SMS;
inline int ggnn_colsum_blocks(int rows) {
  const int b = (rows + 63) / 64;
  return b < GGNN_COLSUM_MAX_BLOCKS ? b : GGNN_COLSUM_MAX_BLOCKS;
}
int launch_ggnn_bias_grad(const float* x, int rows, int N, float* partial, float* out, cudaStream_t stream);

// ---- rgnn_rgin_backward (rgin_backward.cu) ----
// y[0:n] = act(x[0:n])  (n % 4 == 0)
int launch_rgin_act(const float* x, long n, int act, float* y, cudaStream_t stream);
// out [rows, width]: rows < valid = g act'(x) (act LINEAR: g; x unread), divided by the mean / sqrt_n divisor of v when agg
// asks for it (seg_off: all incoming edges of v); rows >= valid zero.  out may be g or x.
struct RginGradParams {
  long rows = 0, valid = 0;
  int width = 0, act = RGNN_ACT_LINEAR, agg = RGNN_AGG_SUM;
  const int32_t* seg_off = nullptr;
  const float* g = nullptr;
  const float* x = nullptr;
  float* out = nullptr;
};
int launch_rgin_act_grad(const RginGradParams& p, cudaStream_t stream);
// out [V, D] = sum over l in order of dq [V, L, D]
int launch_rgin_type_sum(const float* dq, int V, int L, int D, float* out, cudaStream_t stream);

// ---- rgnn_rgdcn_backward (rgdcn_backward.cu) ----
// One warp per target row v < V: rows < Vt write dS [V, L, D] and overwrite the pre-activations P with dP; rows >= Vt zero
// their dS rows.  P holds L * C blocks of K * K floats per target; W[v, l, c] is block v * L * C + l * st_type + c * st_chan
// (full state: the forward's [Vt, L, C, K, K], st_type = C, st_chan = 1; per channel: [Vt, C, L, K, K], st_type = 1,
// st_chan = L).
struct RgdcnBwdParams {
  int V = 0, Vt = 0, L = 1, D = 0, K = 0, C = 1, act = RGNN_ACT_LINEAR, agg = RGNN_AGG_SUM;
  int st_type = 1, st_chan = 1;
  const int32_t* seg_off = nullptr; const int32_t* e_src = nullptr; const int32_t* e_type = nullptr;
  const float* h = nullptr;            // [V, D]   this timestep's input
  const float* grad_out = nullptr;     // [Vt, D]
  const float* num_incoming = nullptr; // [L, scale_ld] or NULL
  int scale_ld = 0;
  float* P = nullptr;                  // [Vt, L * C, K * K]  pre-activations in, dP out
  float* dS = nullptr;                 // [V, L, D]
};
int launch_rgdcn_bwd_target(const RgdcnBwdParams& p, cudaStream_t stream);
// out [rows, KK] = sum over c in order of dp [rows, C, KK]
int launch_rgdcn_chan_sum(const float* dp, long rows, int C, int KK, float* out, cudaStream_t stream);

}  // namespace rgnn
