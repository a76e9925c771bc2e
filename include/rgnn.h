/*
 * rgnn.h -- C ABI of the H100-native relational message-passing engine (librgnn.so).
 *
 * The reference (microsoft/tf-gnn-samples) has no FFI: its boundary is the Python call
 * convention  Sparse_Graph_Model._apply_gnn_layer(node_representations, adjacency_lists,
 * type_to_num_incoming_edges, num_timesteps)  (models/sparse_graph_model.py:204-225), served by
 * gnns.sparse_<x>_layer(...) (gnns/__init__.py:1-7).  Each rgnn_<x>_forward below is what a
 * ctypes binding of that layer function calls; the argument lists mirror the keyword
 * arguments the model adapters pass (models/<x>_model.py), plus explicit weight pointers
 * (the reference creates its weights inside the layer function under a tf.variable_scope).
 *
 * Conventions
 *   return    0 = OK, negative = error (RGNN_E_*); message via rgnn_last_error() (thread-local).
 *             Nothing throws across the ABI, nothing calls exit().
 *   memory    every data pointer is a DEVICE pointer owned by the caller (16-byte aligned,
 *             row-major fp32 / int32); "host array" arguments are small host-side tables
 *             (pointer lists, sizes).  The library borrows pointers for the duration of the
 *             call only.  Plans own their index buffers.
 *   async     all work is enqueued on `stream` (a cudaStream_t passed as void*); forwards
 *             make no hidden synchronisation and are CUDA-Graph capturable.  Calls that synchronise
 *             (and return RGNN_E_INVALID, recording nothing, on a capturing stream): rgnn_plan_create /
 *             _create_ex without RGNN_PLAN_DEFERRED_CHECK, rgnn_plan_status (on the creation stream).
 *             rgnn_halo_plan_create also synchronises, and rgnn_weight_cache_clear /
 *             rgnn_set_weight_cache(0) call cudaFree: never call them during a capture.
 *   capture   run eagerly once before capturing: every layer with the weight cache on (a cache miss
 *             during capture is an error), and the first backward on a plan (rgnn_rgcn_backward /
 *             rgnn_film_backward / rgnn_rgat_backward / rgnn_ggnn_backward / rgnn_rgin_backward /
 *             rgnn_rgdcn_backward / rgnn_edge_aggregate_backward build the plan's reverse index then; inside a capture they
 *             return RGNN_E_INVALID).  A plan built with RGNN_PLAN_DEFERRED_CHECK inside a capture is
 *             filled only when the graph is replayed: call rgnn_plan_status after a replay.  A graph
 *             captured with the weight cache on reads the cached images: rgnn_weight_cache_clear (and
 *             rgnn_set_weight_cache(0)) frees them, so such a graph must not be replayed afterwards.
 *   threads   re-entrant on distinct plans/streams; one plan must not be used concurrently by two host
 *             threads.  A plan may be used on streams other than its creation stream: order them after
 *             the build (a deferred build is still running on the creation stream; a validated one has
 *             finished).  rgnn_plan_destroy frees the plan stream-ordered on the CREATION stream: before
 *             calling it, make that stream wait (event) for the work queued on every other stream that
 *             uses the plan, or the memory may be handed to the next allocation (the next batch's plan)
 *             while that work still reads it.  The Python GraphPlan does both itself.
 *   layouts   node states [V, D] fp32 row-major, D % 4 == 0; adjacency lists int32 [E_l, 2]
 *             (col 0 = source, col 1 = target: gnns/rgcn.py:85-86); in-degrees fp32 [L, V]
 *             (tasks/sparse_graph_task.py:145); weights in Keras orientation kernel[in, out]
 *             (y = x . kernel) so reference checkpoints load without transposition.
 */
#ifndef RGNN_H_
#define RGNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define RGNN_API __attribute__((visibility("default")))
#else
#define RGNN_API
#endif

#define RGNN_VERSION 200          /* 0.2.0 */
#define RGNN_MAX_EDGE_TYPES 64
#define RGNN_MAX_MLP_LAYERS 8
#define RGNN_MAX_STATE_DIM 512    /* per-row register tile of the segment kernels */
#define RGNN_MAX_WORLD 16         /* ranks of one node-range partition (one NVSwitch domain) */
#define RGNN_PEER_HANDLE_BYTES 64 /* sizeof(cudaIpcMemHandle_t) */

/* error codes */
#define RGNN_OK 0
#define RGNN_E_INVALID (-1)       /* bad argument (NULL, misaligned, dim % 4 != 0, unknown enum ...) */
#define RGNN_E_CUDA (-2)          /* CUDA runtime error; message carries cudaGetErrorString */
#define RGNN_E_WORKSPACE (-3)     /* workspace too small */
#define RGNN_E_UNSUPPORTED (-4)   /* valid in the reference but outside this build's limits */

/* utils/utils.py:36-58 get_activation (names lower-cased there) */
enum rgnn_activation {
  RGNN_ACT_LINEAR = 0, RGNN_ACT_TANH = 1, RGNN_ACT_RELU = 2, RGNN_ACT_LEAKY_RELU = 3,
  RGNN_ACT_ELU = 4, RGNN_ACT_SELU = 5, RGNN_ACT_GELU = 6
};
/* utils/utils.py:23-33 get_aggregation_function */
enum rgnn_aggregation { RGNN_AGG_SUM = 0, RGNN_AGG_MAX = 1, RGNN_AGG_MEAN = 2, RGNN_AGG_SQRT_N = 3 };
/* utils/utils.py:10-20 get_gated_unit (LSTM is unusable as the reference calls it: ggnn.py:92) */
enum rgnn_cell { RGNN_CELL_RNN = 0, RGNN_CELL_GRU = 1 };
enum rgnn_layer_kind {
  RGNN_LAYER_RGCN = 0, RGNN_LAYER_GGNN = 1, RGNN_LAYER_RGAT = 2, RGNN_LAYER_FILM = 3,
  RGNN_LAYER_EDGE_MLP = 4, RGNN_LAYER_RGIN = 5, RGNN_LAYER_RGCN_BACKWARD = 6,
  RGNN_LAYER_RGDCN = 7,  /* rgnn_workspace_bytes: pass channel_dim as mlp_layers */
  RGNN_LAYER_FILM_BACKWARD = 8, RGNN_LAYER_RGAT_BACKWARD = 9, RGNN_LAYER_GGNN_BACKWARD = 10,
  RGNN_LAYER_RGIN_BACKWARD = 11,
  RGNN_LAYER_RGDCN_BACKWARD = 12  /* rgnn_workspace_bytes: pass channel_dim as mlp_layers */
};

typedef struct rgnn_plan rgnn_plan_t;
typedef struct rgnn_halo_plan rgnn_halo_plan_t;

RGNN_API int rgnn_version(void);
RGNN_API const char* rgnn_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py "gpu_launches") */
RGNN_API int64_t rgnn_launch_count(void);

/*
 * Plan = the batch's graph structure in the layout the kernels want, built once per batch and
 * reused by every layer and timestep (replaces the per-layer tf.concat of targets + unsorted
 * segment ids: gnns/rgcn.py:76-78,108-112).  Contents (device): CSR by target over ALL edge
 * types, incoming edges of a node sorted by (type, original position) -- a stable sort, so
 * every reduction order is deterministic.
 *   adjacency_lists : host array of L device pointers, each int32 [E_l, 2]
 *   num_edges       : host array [L] (E_l may be 0: tasks/ppi_task.py:246-249)
 */
RGNN_API int rgnn_plan_create(rgnn_plan_t** out, int32_t num_nodes, int32_t num_edge_types,
                     const int32_t* const* adjacency_lists, const int64_t* num_edges, void* stream);
/* Same, with flags.  RGNN_PLAN_DEFERRED_CHECK: do not synchronise; the index-range check result stays on the
 * device until rgnn_plan_status() (which synchronises the creation stream) is called.  Out-of-range ids are
 * clamped to node 0 inside the plan, so later kernels stay memory-safe either way. */
#define RGNN_PLAN_DEFERRED_CHECK 1
RGNN_API int rgnn_plan_create_ex(rgnn_plan_t** out, int32_t num_nodes, int32_t num_edge_types,
                        const int32_t* const* adjacency_lists, const int64_t* num_edges, int flags, void* stream);
RGNN_API int rgnn_plan_status(const rgnn_plan_t* plan);
/* Sharded execution (one rank of a node-range partition: owned nodes first, halo nodes after them): declare that only
 * rows [0, num_targets) are targets whose outputs are wanted.  The edge stage then reduces only those rows and the
 * TARGET-side node-level work of the layers (FiLM's gamma/beta GEMM, GGNN's cell, RGDCN's dynamic kernels, RGIN's
 * aggregation MLP and layer norm) runs on them only; source-side transforms still cover all V rows.  Output rows
 * >= num_targets are left untouched; layers must be called with num_timesteps == 1 and rgnn_rgcn_stack_forward with
 * num_layers == 1 (halo states are refreshed by the caller's exchange between steps).  Default: num_targets = V. */
RGNN_API int rgnn_plan_set_num_targets(rgnn_plan_t* plan, int32_t num_targets);
RGNN_API int rgnn_plan_destroy(rgnn_plan_t* plan);
RGNN_API int32_t rgnn_plan_num_nodes(const rgnn_plan_t* plan);
RGNN_API int32_t rgnn_plan_num_edge_types(const rgnn_plan_t* plan);
RGNN_API int64_t rgnn_plan_num_edges(const rgnn_plan_t* plan);       /* M = sum_l E_l */
/* Copy the plan's arrays into caller DEVICE buffers (any may be NULL): seg_off [V+1],
 * e_src [M], e_type [M], e_orig [M] (position in the type-major concatenation of the inputs). */
RGNN_API int rgnn_plan_export(const rgnn_plan_t* plan, int32_t* seg_off, int32_t* e_src, int32_t* e_type,
                     int32_t* e_orig, void* stream);

/* Static-weight mode (inference / benchmarking), off by default.  The tensor-core GEMM consumes the
 * weights as pre-swizzled TF32 hi/lo shared-memory images; normally they are rebuilt from the caller's
 * kernels on every forward.  With the cache on, images are built once per distinct (weight pointers,
 * shape, tiling) and reused; the caller must call rgnn_weight_cache_clear() after changing cached weights
 * in place.  A cache miss inside CUDA-graph capture is an error (run the layer once eagerly first).
 * The key holds device ADDRESSES, not contents: a caller that frees a cached weight and later receives the same address for a
 * different weight (a new model in the same process) must call rgnn_weight_cache_clear() in between, or the old images are
 * used silently.  The Python binding does this itself (it tracks the owning tensor's lifetime and version per address). */
RGNN_API int rgnn_set_weight_cache(int enable);
RGNN_API int rgnn_weight_cache_clear(void);

/* Upper bound of the scratch a forward of `layer_kind` needs.  mlp_layers = number of kernels
 * in the widest edge/aggregation MLP (0 if none).  The bound assumes every MLP layer is at most max(2 * d_in, d_out)
 * wide (true of the reference's MLPs, whose hidden layers are d_out wide); rgnn_edge_mlp_forward and rgnn_rgin_forward
 * refuse a wider layer with RGNN_E_UNSUPPORTED before enqueueing anything.
 *
 * Workspace contract of every call that takes one: the workspace needs 16-byte alignment only (carve-outs are aligned
 * relative to its start), its contents on entry are never read, and the call writes nothing past workspace_bytes.  A call
 * that returns RGNN_E_WORKSPACE (a NULL workspace counts as 0 bytes) has written no output and nothing outside the
 * workspace; it may already have enqueued kernels that write inside the first workspace_bytes of it (the Edge-MLP, RGIN and
 * backward paths carve their scratch as they go), so the workspace's contents are undefined afterwards. */
RGNN_API size_t rgnn_workspace_bytes(const rgnn_plan_t* plan, int layer_kind, int32_t d_in, int32_t d_out,
                            int32_t mlp_layers);

/* ---- gnns/rgcn.py:8-117  sparse_rgcn_layer ------------------------------------------------
 * edge_weights: host array of L device pointers, kernel [d_in * (1 + use_both), d_out].
 * num_incoming: [L, V] fp32 or NULL when normalize == 0.  num_timesteps > 1 needs d_in == d_out. */
RGNN_API int rgnn_rgcn_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                      const float* const* edge_weights, const float* num_incoming,
                      int activation, int aggregation, int normalize_by_num_incoming,
                      int use_both_source_and_target, int num_timesteps,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_rgcn_layer with source-only messages (use_both_source_and_target = 0):
 * the gradients TensorFlow autodiff produces for gnns/rgcn.py:84-114 (models/sparse_graph_model.py:253-260).
 *   out       forward output [V, d_out] (act' is evaluated from it; gelu recomputes the pre-activation)
 *   grad_out  dLoss/d out [V, d_out]
 *   grad_node_embeddings [V, d_in] or NULL; grad_edge_weights: host array of L device pointers [d_in, d_out] or NULL
 * 'max' aggregation is not differentiated in this build (RGNN_E_UNSUPPORTED).  The first backward on a plan builds
 * a reverse (by-source) index inside it (not thread-safe).  Workspace: rgnn_workspace_bytes(RGNN_LAYER_RGCN_BACKWARD). */
RGNN_API int rgnn_rgcn_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                       const float* const* edge_weights, const float* num_incoming,
                       int activation, int aggregation, int normalize_by_num_incoming,
                       const float* out, const float* grad_out,
                       float* grad_node_embeddings, float* const* grad_edge_weights,
                       void* workspace, size_t workspace_bytes, void* stream);

/* graph_num_layers x sparse_rgcn_layer in one call -- the GNN loop of
 * Sparse_Graph_Model.__build_graph_propagation_model (models/sparse_graph_model.py:176-191) without the scaffold's
 * dropout / residual / inter-layer Dense.  edge_weights: host array of num_layers * L pointers (layer-major),
 * every kernel [d, d]; the layers share activation / aggregation / normalisation like RGCN_Model does.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_RGCN, d, d, 0) + 2 * (V * d * 4 + 256) bytes (two inter-layer buffers of
 * [V, d] floats, each rounded up to 256 bytes, then one layer's scratch); less returns RGNN_E_WORKSPACE. */
RGNN_API int rgnn_rgcn_stack_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d, int32_t num_layers,
                            const float* const* edge_weights, const float* num_incoming,
                            int activation, int aggregation, int normalize_by_num_incoming,
                            float* out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- gnns/ggnn.py:8-95  sparse_ggnn_layer --------------------------------------------------
 * cell_kernel [d, 3d] (GRU, gates z|r|h) or [d, d] (RNN); cell_recurrent_kernel same shape;
 * cell_bias [3d] / [d].  d_in must equal d_out (the cell state is the node state: ggnn.py:92). */
RGNN_API int rgnn_ggnn_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                      const float* const* edge_weights, const float* cell_kernel,
                      const float* cell_recurrent_kernel, const float* cell_bias,
                      int cell_kind, int activation, int aggregation, int num_timesteps,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_ggnn_layer (ggnn.py:76-93, Keras TF-1.13 GRU / SimpleRNN cell): the gradients
 * TensorFlow autodiff produces.  Gradients are written, not accumulated.  No forward state is needed: the call recomputes the
 * aggregate m and the cell's pre-activations from its inputs, and builds no per-edge tensor.
 *   node_embeddings [V, d]: this timestep's INPUT; weights as rgnn_ggnn_forward (cell_bias 16-byte aligned too)
 *   grad_out [num_targets, d] (rows [0, num_targets) of the plan, rgnn_plan_set_num_targets)
 *   grad_node_embeddings [V, d] covers EVERY local row (halo rows included: what rgnn_halo_exchange_backward consumes) or
 *   NULL, and must not alias node_embeddings or grad_out; grad_edge_weights: host array of L device pointers [d, d] or NULL;
 *   grad_cell_kernel / grad_cell_recurrent_kernel [d, 3d] (GRU) / [d, d] (RNN) or NULL; grad_cell_bias [3d] / [d] or NULL.
 * 'max' aggregation: RGNN_E_UNSUPPORTED.  Every argument is checked and the workspace sized before anything is enqueued.
 * The first backward on a plan builds its reverse index (as rgnn_rgcn_backward; not inside a capture).  Two identical calls
 * are bit-identical (no atomics: every output has one writer, every sum a fixed order).
 * Several timesteps are the caller's loop: run the forward with num_timesteps = 1 per timestep keeping each input, call
 * this from the last timestep down (grad_out of step t = grad_node_embeddings of step t + 1), and add the shared weights'
 * gradients of the steps.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_GGNN_BACKWARD, d, d, 0): with V = num_nodes, L = num_edge_types,
 * (V L d + 11 V d + 792 d + (L + 3) d^2 + 2228224) floats plus the weight-image scratch of the forward's bound. */
RGNN_API int rgnn_ggnn_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d,
                       const float* const* edge_weights, const float* cell_kernel, const float* cell_recurrent_kernel,
                       const float* cell_bias, int cell_kind, int activation, int aggregation,
                       const float* grad_out, float* grad_node_embeddings, float* const* grad_edge_weights,
                       float* grad_cell_kernel, float* grad_cell_recurrent_kernel, float* grad_cell_bias,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- gnns/rgat.py:9-141  sparse_rgat_layer -------------------------------------------------
 * attention: host array of L device pointers [2 * d_out]; head k uses [k*2d, (k+1)*2d),
 * first d for the source, next d for the target (rgat.py:110-111), d = d_out / num_heads. */
RGNN_API int rgnn_rgat_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                      const float* const* edge_weights, const float* const* attention,
                      int num_heads, int activation, int num_timesteps,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_rgat_layer (rgat.py:83-139): the gradients TensorFlow autodiff produces.
 * Gradients are written, not accumulated.  No forward state is needed: the call recomputes h . W_l, the per-head scores
 * and the softmax from its inputs, and builds no per-edge tensor.
 *   node_embeddings [V, d_in]: this timestep's INPUT; attention: as rgnn_rgat_forward (16-byte aligned)
 *   grad_out [num_targets, d_out] (rows [0, num_targets) of the plan, rgnn_plan_set_num_targets)
 *   grad_node_embeddings [V, d_in] covers EVERY local row (halo rows included: what rgnn_halo_exchange_backward consumes)
 *   or NULL; grad_edge_weights: host array of L device pointers [d_in, d_out] or NULL; grad_attention: host array of L
 *   device pointers [2 * d_out] or NULL.
 * d_out > RGNN_MAX_STATE_DIM and per-head dims d_out / num_heads that are not multiples of 4 return RGNN_E_UNSUPPORTED;
 * num_heads must divide d_out.  Every argument is checked and the workspace sized before anything is enqueued.  The first
 * backward on a plan builds its reverse index (as rgnn_rgcn_backward; not inside a capture).  Two identical calls are
 * bit-identical (no atomics: every output has one writer, every sum a fixed order).
 * Several timesteps are the caller's loop: run the forward with num_timesteps = 1 per timestep keeping each input, call
 * this from the last timestep down (grad_out of step t = grad_node_embeddings of step t + 1), and add the shared weights'
 * gradients of the steps.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_RGAT_BACKWARD, d_in, d_out, 0), a bound for every head count: with
 * V = num_nodes, L = num_edge_types, D = d_out, (3 V L D + 2 V D + 528 L D + L d_in D + 2228224) floats plus the
 * weight-image scratch of the forward's bound. */
RGNN_API int rgnn_rgat_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                       const float* const* edge_weights, const float* const* attention, int num_heads, int activation,
                       const float* grad_out, float* grad_node_embeddings, float* const* grad_edge_weights,
                       float* const* grad_attention, void* workspace, size_t workspace_bytes, void* stream);

/* ---- gnns/gnn_film.py:8-122  sparse_gnn_film_layer -----------------------------------------
 * film_weights: L pointers, kernel [d_in, 2*d_out] (gamma = cols [0,d), beta = cols [d,2d)).
 * ln_gamma / ln_beta: [num_timesteps, d_out] (one LayerNorm scope per timestep: gnn_film.py:120). */
RGNN_API int rgnn_film_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                      const float* const* edge_weights, const float* const* film_weights,
                      const float* num_incoming, const float* ln_gamma, const float* ln_beta,
                      int activation, int aggregation, int normalize_by_num_incoming, int num_timesteps,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_gnn_film_layer (gnn_film.py:85-120): the gradients TensorFlow autodiff produces.
 * Gradients are written, not accumulated.  No forward state is needed: the call recomputes h . W_l, h . F_l and the
 * aggregate from its inputs.
 *   node_embeddings [V, d_in]: this timestep's INPUT; ln_gamma / ln_beta: this timestep's [d_out]
 *   grad_out [num_targets, d_out] (rows [0, num_targets) of the plan, rgnn_plan_set_num_targets)
 *   grad_node_embeddings [V, d_in] covers EVERY local row (halo rows included: what rgnn_halo_exchange_backward consumes)
 *   or NULL; grad_edge_weights / grad_film_weights: host arrays of L device pointers ([d_in, d_out] / [d_in, 2 d_out]) or
 *   NULL; grad_ln_gamma / grad_ln_beta [d_out] or NULL.
 * 'max' aggregation: RGNN_E_UNSUPPORTED, as is d_out > RGNN_MAX_STATE_DIM.  Every argument is checked and the workspace
 * sized before anything is enqueued.  The first backward on a plan builds its reverse index (as rgnn_rgcn_backward; not
 * inside a capture).  Two identical calls are bit-identical (every output has one writer, every sum a fixed order).
 * Several timesteps are the caller's loop: run the forward with num_timesteps = 1 per timestep keeping each input, call
 * this from the last timestep down (grad_out of step t = grad_node_embeddings of step t + 1), and add the shared weights'
 * gradients of the steps.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_FILM_BACKWARD, d_in, d_out, 0). */
RGNN_API int rgnn_film_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                       const float* const* edge_weights, const float* const* film_weights, const float* num_incoming,
                       const float* ln_gamma, const float* ln_beta, int activation, int aggregation,
                       int normalize_by_num_incoming, const float* grad_out, float* grad_node_embeddings,
                       float* const* grad_edge_weights, float* const* grad_film_weights, float* grad_ln_gamma,
                       float* grad_ln_beta, void* workspace, size_t workspace_bytes, void* stream);

/* ---- gnns/gnn_edge_mlp.py:7-122  sparse_gnn_edge_mlp_layer ---------------------------------
 * mlp_kernels: host array of L * (num_edge_hidden_layers + 1) device pointers, type-major;
 * layer j of every type has shape [mlp_dims[j], mlp_dims[j+1]]; mlp_dims host [layers + 1],
 * mlp_dims[0] = d_in * (1 + use_target_state_as_input), mlp_dims[last] = d_out, every mlp_dims[j >= 1] at most
 * max(2 * d_in, d_out) (RGNN_E_UNSUPPORTED otherwise; the same limit holds for both MLPs of rgnn_rgin_forward).
 * Hidden activation is ELU regardless of `activation` (gnn_edge_mlp.py:76). */
RGNN_API int rgnn_edge_mlp_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                          const float* const* mlp_kernels, const int32_t* mlp_dims, int num_edge_hidden_layers,
                          const float* num_incoming, const float* ln_gamma, const float* ln_beta,
                          int activation, int aggregation, int normalize_by_num_incoming,
                          int use_target_state_as_input, int num_timesteps,
                          float* out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- gnns/rgin.py:7-142  sparse_rgin_layer -------------------------------------------------
 * num_edge_mlp_hidden_layers < 0  <=>  None (messages are the raw source states, no activation).
 * num_aggr_mlp_hidden_layers < 0  <=>  None.  aggr_kernels: host array of (layers+1) pointers,
 * aggr_dims host [layers + 2].  Edge-MLP hidden activation = `activation` (rgin.py:95). */
RGNN_API int rgnn_rgin_forward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                      const float* const* edge_mlp_kernels, const int32_t* edge_mlp_dims,
                      int num_edge_mlp_hidden_layers,
                      const float* const* aggr_kernels, const int32_t* aggr_dims,
                      int num_aggr_mlp_hidden_layers,
                      const float* ln_gamma, const float* ln_beta,
                      int activation, int aggregation, int use_target_state_as_input, int num_timesteps,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_rgin_layer with source-only messages (rgin.py:103-139, use_target_state_as_input = 0:
 * the default of every reference config): the gradients TensorFlow autodiff produces.  Gradients are written, not
 * accumulated.  No forward state is needed: the call recomputes the edge MLP on the node rows (a message depends on its
 * source and type only), the aggregate and the aggregation MLP from its inputs, and builds no per-edge tensor.
 *   node_embeddings [V, d_in]: this timestep's INPUT; the MLP tables and dims as rgnn_rgin_forward (either MLP may be None,
 *   with the same width limits); ln_gamma / ln_beta: this timestep's [d_out]
 *   grad_out [num_targets, d_out] (rows [0, num_targets) of the plan, rgnn_plan_set_num_targets)
 *   grad_node_embeddings [V, d_in] covers EVERY local row (halo rows included: what rgnn_halo_exchange_backward consumes) or
 *   NULL, and must not alias node_embeddings or grad_out; grad_edge_mlp_kernels: host array of L * n_e device pointers
 *   (type-major, as the forward's table) or NULL; grad_aggr_kernels: host array of n_a device pointers or NULL;
 *   grad_ln_gamma / grad_ln_beta [d_out] or NULL.  (n_e, n_a = number of kernels of the edge / aggregation MLP.)
 * use_target_state_as_input = 1, 'max' aggregation and d_out > RGNN_MAX_STATE_DIM: RGNN_E_UNSUPPORTED.  Every argument is
 * checked and the workspace sized before anything is enqueued.  The first backward on a plan builds its reverse index (as
 * rgnn_rgcn_backward; not inside a capture).  Two identical calls are bit-identical (no atomics: every output has one
 * writer, every sum a fixed order).
 * Several timesteps are the caller's loop: run the forward with num_timesteps = 1 per timestep keeping each input, call
 * this from the last timestep down (grad_out of step t = grad_node_embeddings of step t + 1), and add the shared weights'
 * gradients of the steps.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_RGIN_BACKWARD, d_in, d_out, max(n_e, n_a)): with V = num_nodes,
 * L = num_edge_types, dm = max(2 d_in, d_out), nl = max(n_e, n_a, 1),
 * (2 nl V L dm + (2 nl + 2) V dm + 528 d_out + L dm^2 + 2228224) floats plus the weight-image scratch of the forward's bound. */
RGNN_API int rgnn_rgin_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d_in, int32_t d_out,
                       const float* const* edge_mlp_kernels, const int32_t* edge_mlp_dims, int num_edge_mlp_hidden_layers,
                       const float* const* aggr_kernels, const int32_t* aggr_dims, int num_aggr_mlp_hidden_layers,
                       const float* ln_gamma, const float* ln_beta, int activation, int aggregation,
                       int use_target_state_as_input, const float* grad_out, float* grad_node_embeddings,
                       float* const* grad_edge_mlp_kernels, float* const* grad_aggr_kernels, float* grad_ln_gamma,
                       float* grad_ln_beta, void* workspace, size_t workspace_bytes, void* stream);

/* gnns/rgdcn.py:8-171 -- relational graph DYNAMIC convolution: the state is split into num_channels channels of
 * K = d / num_channels; message of edge (u -> v, type l), channel c:  h_u[c,:] . W[v,l,c]  with the K x K kernel
 * W[v,l,c] = reshape(act(F_{l,c} . x_v)), x_v = h_v (use_full_state) or h_v[c,:]; then 1/(c+1e-7) scaling, aggregation over
 * all types, activation.  channel_weights: host array of L*num_channels device pointers, entry l*num_channels + c =
 * F_{l,c} [d or K, K*K] (Keras Dense kernel; tie_channel_weights = the same pointer for every c).  K must be a power of
 * two in [4, 128], d <= 512.  For sum / mean / sqrt_n the per-(target, type) source rows are summed before ONE matvec per
 * channel (the kernel depends on the target only); max applies it per edge. */
RGNN_API int rgnn_rgdcn_forward(const rgnn_plan_t* plan, const float* h, int32_t d, int32_t num_channels,
                       const float* const* channel_weights, int use_full_state, const float* num_incoming,
                       int activation, int aggregation, int normalize, int num_timesteps, float* out,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Backward of ONE timestep of sparse_rgdcn_layer (rgdcn.py:116-165; all four variants, sum / mean / sqrt_n, every
 * activation): the gradients TensorFlow autodiff produces.  Gradients are written, not accumulated.  No forward state is
 * needed: the call recomputes the dynamic kernels' pre-activations and the aggregate from its inputs, and builds no
 * per-edge tensor.
 *   node_embeddings [V, d]: this timestep's INPUT; channel_weights, use_full_state, num_incoming, activation, aggregation,
 *   normalize: as rgnn_rgdcn_forward (host array of L * num_channels kernels, type-major, [d or K, K*K] each)
 *   grad_out [num_targets, d] (rows [0, num_targets) of the plan, rgnn_plan_set_num_targets)
 *   grad_node_embeddings [V, d] covers EVERY local row (halo rows included: what rgnn_halo_exchange_backward consumes) or
 *   NULL, and must not alias node_embeddings or grad_out
 *   grad_channel_weights: host array of L * num_channels device pointers laid out like channel_weights, or NULL.
 *   tie_channel_weights = 1 (one kernel per edge type, rgdcn.py:96,105-107): every entry of type l must be the same pointer,
 *   in channel_weights and in grad_channel_weights, and dF_l (the sum over the channels) is written once.  Untied: the
 *   entries of grad_channel_weights must be distinct.  Either violation is refused, naming the argument.
 * Limits are the forward's: K = d / num_channels a power of two in [4, 128], num_channels <= RGNN_MAX_EDGE_TYPES, 16-byte
 * alignment; d > RGNN_MAX_STATE_DIM and 'max' aggregation: RGNN_E_UNSUPPORTED.  Every argument is checked and the workspace
 * sized before anything is enqueued.  The first backward on a plan builds its reverse index (as rgnn_rgcn_backward; not
 * inside a capture).  Two identical calls are bit-identical (no atomics: every output has one writer, every sum a fixed
 * order).
 * Several timesteps are the caller's loop: run the forward with num_timesteps = 1 per timestep keeping each input, call
 * this from the last timestep down (grad_out of step t = grad_node_embeddings of step t + 1), and add the shared weights'
 * gradients of the steps.
 * Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_RGDCN_BACKWARD, d, d, K): with V = num_nodes, Vt = num_targets,
 * L = num_edge_types, C = d / K, Q = min(L C, 64) K^2,
 * (Vt L d K + 2 V L d + Vt d + Vt L K^2 + d Q + 2 (Q + 128)(d + 128) + 2163712) floats plus the weight-image scratch of the
 * forward's bound, 2 (4 d + 64)(4 L d + 4 d + 512) floats, plus 8192 bytes.  No term grows with the number of edges. */
RGNN_API int rgnn_rgdcn_backward(const rgnn_plan_t* plan, const float* node_embeddings, int32_t d, int32_t num_channels,
                        const float* const* channel_weights, int use_full_state, int tie_channel_weights,
                        const float* num_incoming, int activation, int aggregation, int normalize,
                        const float* grad_out, float* grad_node_embeddings, float* const* grad_channel_weights,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- one large graph over several GPUs: node-range partition + halo exchange (SURVEY.md 8e) --------------------------
 * The reference is single-device; this is the multi-GPU form of ITS batch (tasks/varmisuse_task.py:451-538 packs up to
 * 100k nodes per batch): rank r of `world` owns the nodes [cuts[r], cuts[r+1]) and every edge whose TARGET it owns, so the
 * segment reductions / softmax / layer norm / GRU of every layer stay local; before each layer the states of the remote
 * SOURCE nodes ("halo") are refreshed.  One process per GPU; weights are replicated.
 *
 * rgnn_halo_plan_create: adjacency_lists hold GLOBAL node ids (device, int32 [E_l, 2]); edges whose target another rank
 * owns are dropped, so every rank may pass the same lists or only its own shard.  Built on the device (order-preserving
 * select, radix sort + unique of the remote sources, renumbering).  Local numbering: owned node g -> g - cuts[rank];
 * halo nodes follow, sorted by global id (hence grouped by owner).  rgnn_halo_plan_graph() is the ordinary plan over the
 * local ids with num_targets = the owned rows: pass it to any rgnn_<x>_forward with node states [n_own + n_halo, d]
 * (num_timesteps = 1 per call; call rgnn_halo_exchange between steps).  Synchronises the stream (it sizes buffers). */
RGNN_API int rgnn_halo_plan_create(rgnn_halo_plan_t** out, int32_t rank, int32_t world, const int64_t* cuts /* host [world+1] */,
                          int32_t num_edge_types, const int32_t* const* adjacency_lists, const int64_t* num_edges,
                          void* stream);
RGNN_API int rgnn_halo_plan_destroy(rgnn_halo_plan_t* plan);
RGNN_API int32_t rgnn_halo_plan_num_own(const rgnn_halo_plan_t* plan);
RGNN_API int32_t rgnn_halo_plan_num_halo(const rgnn_halo_plan_t* plan);
RGNN_API int64_t rgnn_halo_plan_num_edges(const rgnn_halo_plan_t* plan, int32_t edge_type);   /* kept edges of one type */
RGNN_API rgnn_plan_t* rgnn_halo_plan_graph(rgnn_halo_plan_t* plan);                            /* owned by the halo plan */
/* Copies into caller DEVICE buffers (any may be NULL): halo_global / halo_owner / halo_row [n_halo] (global id, owning rank,
 * row inside the owner's state buffer) and the renumbered adjacency lists (host array of L device pointers, [E_l, 2]). */
RGNN_API int rgnn_halo_plan_export(const rgnn_halo_plan_t* plan, int32_t* halo_global, int32_t* halo_owner, int32_t* halo_row,
                          int32_t* const* local_adjacency_lists, void* stream);
/* Peer memory.  Every rank keeps TWO state buffers (layer t reads buffer t % 2 and writes its owned rows into the other
 * one) of [n_own + n_halo, d] floats, owned rows first, plus one flag array uint32[world], in memory that the other ranks
 * have mapped into their address space (rgnn_peer_* below, or any other mechanism: these are plain device pointers).
 * peer_states0/1 and peer_flags are host arrays of `world` device pointers valid IN THIS PROCESS; entry [rank] is this
 * rank's own memory.  The flag arrays must start zeroed. */
RGNN_API int rgnn_halo_plan_attach(rgnn_halo_plan_t* plan, void* const* peer_states0, void* const* peer_states1,
                          void* const* peer_flags);
/* Refresh rows [n_own, n_own + n_halo) of this rank's state buffer `buffer` with the owners' current rows, read straight
 * out of the owners' buffers over NVLink (one kernel, pull-based: no packing, no send side).  Collective: every rank calls
 * it the same number of times, in the same order; the kernel contains the cross-rank barrier ("every rank's owned rows of
 * this buffer are final") as system-scope flags, and keeps its epoch on the device, so a captured CUDA graph can be
 * replayed.  A peer that never arrives faults the kernel after 10 s instead of hanging the GPU. */
RGNN_API int rgnn_halo_exchange(rgnn_halo_plan_t* plan, int buffer, int32_t d, void* stream);
/* The same exchange off the caller's critical path: the pull is forked onto a stream of the plan (ordered after everything
 * enqueued on `stream` so far) and is NOT joined here.  The next rgnn_<x>_forward on rgnn_halo_plan_graph() joins it right
 * before its first kernel that reads halo rows -- GNN-FiLM runs its target-side gamma / beta GEMM (owned rows only) first, so
 * that GEMM overlaps the transfer over NVLink.  Capturable into a CUDA graph (fork / join through events). */
RGNN_API int rgnn_halo_exchange_overlapped(rgnn_halo_plan_t* plan, int buffer, int32_t d, void* stream);

/* Training over the partition: the transpose of rgnn_halo_exchange.  A rank's layers produce gradients for its local rows
 * [n_own + n_halo, d]; the rows >= n_own belong to other ranks and must be ADDED to their owners' rows.  The same
 * peer-memory design carries them back, with no host-side index and no NCCL call on the data path.
 *
 * rgnn_halo_plan_attach_grad: like rgnn_halo_plan_attach, for the backward direction.  Every rank keeps TWO gradient
 * buffers of [n_own + n_halo, d] floats (16-byte aligned; consecutive backward exchanges alternate them, as consecutive
 * forward exchanges alternate the state buffers), a flag array uint32[world] that must start zeroed and must NOT be the
 * forward exchange's (the two barriers never satisfy each other), and a halo list of int32 [4 + 2 * n_halo] (16-byte
 * aligned).  The call writes this rank's halo list there ([0] = n_halo, [4, 4 + n_halo) = owners, [4 + n_halo,
 * 4 + 2 n_halo) = rows in the owners' buffers) and synchronises.  All pointer arrays are host arrays of `world` device
 * pointers valid in this process, entry [rank] = this rank's own memory.
 *
 * rgnn_halo_plan_build_reverse: once EVERY rank has returned from rgnn_halo_plan_attach_grad (a host-side barrier, e.g.
 * torch.distributed.barrier), each rank reads its peers' published lists and builds on the device the reverse index:
 * for every owned row, the (peer, row of that peer's gradient buffer) pairs that hold it as a halo row, sorted by (owned
 * row, peer rank).  Synchronises `stream`; returns RGNN_E_INVALID, recording nothing, on a capturing stream.  Run it
 * eagerly once per batch (per halo plan), before any capture.  rgnn_halo_plan_num_reverse: number of pairs (-1 before
 * the build); rgnn_halo_plan_export_reverse copies the index into caller DEVICE buffers (any may be NULL): offsets
 * [n_own + 1], peer and row [num_reverse].
 *
 * rgnn_halo_exchange_backward: grad_own[r] = grad_local[r] + the consumers' gradients of row r, added in ascending peer
 * rank (a fixed order: bit-reproducible, no atomics); a row that no peer consumes is copied bit for bit.  grad_local
 * [n_own + n_halo, d] is read (its halo rows are first copied into this rank's gradient buffer `buffer`, unless
 * grad_local IS that buffer), grad_own [n_own, d] is written.  Collective, with rgnn_halo_exchange's discipline: every
 * rank calls it the same number of times, in the same order, typically in the reverse order of the forward exchanges with
 * the same buffer parity.  Capturable into a CUDA graph once the reverse index exists; its epoch lives on the device.  A
 * peer that never arrives faults the kernel after 10 s.
 *
 * Calling order per batch: rgnn_halo_plan_create, rgnn_halo_plan_attach + rgnn_halo_plan_attach_grad, host barrier,
 * rgnn_halo_plan_build_reverse; then per step: forward = { write owned rows into states(t % 2), rgnn_halo_exchange,
 * layer t } for every layer, backward = { layer t backward on rgnn_halo_plan_graph's local graph,
 * rgnn_halo_exchange_backward(t % 2) } from the last layer down.  Only the halo traffic is handled here: the weight
 * gradients are still summed over the ranks by the caller (an all-reduce; scaffold.all_reduce_gradients_ in Python).
 *
 * Several ranks in one process on one GPU ("virtual ranks", tests): enqueue each rank's work on its own stream, make no
 * call that waits for the device between a rank's exchanges, and keep every rank's exchange kernels co-resident (each
 * launches at most ceil(rows / 128) CTAs of 512 threads, capped at 264 -- rows = n_halo forward, n_own backward; an H100
 * holds 528 such CTAs in all): a rank's CTAs spin until every other rank's first CTA has run.  CUDA loads a kernel at its
 * first launch (lazy module loading, the default) and that load can wait for the running kernels, a spinning exchange
 * included: launch every other kernel of the step once before the ranks' exchanges, and enqueue the ranks phase by phase
 * (every rank's exchange before any rank's next kernel).  rgnn_halo_plan_attach_grad loads the two exchange kernels. */
RGNN_API int rgnn_halo_plan_attach_grad(rgnn_halo_plan_t* plan, void* const* peer_grads0, void* const* peer_grads1,
                               void* const* peer_grad_flags, void* const* peer_halo_lists);
RGNN_API int rgnn_halo_plan_build_reverse(rgnn_halo_plan_t* plan, void* stream);
RGNN_API int64_t rgnn_halo_plan_num_reverse(const rgnn_halo_plan_t* plan);
RGNN_API int rgnn_halo_plan_export_reverse(const rgnn_halo_plan_t* plan, int32_t* offsets, int32_t* peer, int32_t* row,
                                  void* stream);
RGNN_API int rgnn_halo_exchange_backward(rgnn_halo_plan_t* plan, int buffer, int32_t d, const float* grad_local,
                                float* grad_own, void* stream);

/* CUDA-IPC plumbing for the above (one node): allocate zeroed device memory that peers can map, export its 64-byte handle
 * (ship it with any host-side channel, e.g. torch.distributed.all_gather_object), map a peer's allocation. */
RGNN_API int rgnn_peer_alloc(void** ptr, size_t bytes, void* handle_out /* RGNN_PEER_HANDLE_BYTES */);
RGNN_API int rgnn_peer_open(const void* handle, void** ptr);
RGNN_API int rgnn_peer_close(void* ptr);
RGNN_API int rgnn_peer_free(void* ptr);

/* ---- minibatch packing on the device (tasks/ppi_task.py:197-256, tasks/qm9_task.py:200-261) ------------------------
 * The task batchers pack graphs into one block-diagonal graph on the host.  Here a whole data set stays on the device,
 * concatenated in data-set order with GRAPH-LOCAL node ids (CSR over its G graphs and N nodes):
 *   node_offsets     int64 [G + 1], graph g owns the nodes [node_offsets[g], node_offsets[g + 1])
 *   edge_offsets     host array of L device pointers, int64 [G + 1] each: graph g's edges of type l are rows
 *                    [edge_offsets[l][g], edge_offsets[l][g + 1]) of adjacency_lists[l] (int32 [E_l, 2], 8-byte aligned,
 *                    (source, target) local to the graph, in the graph's own order)
 *   num_incoming     fp32 [L, N] (in-degrees as the batcher feeds them)
 *   node_tensors     host array of num_node_tensors device pointers, fp32 [N, node_widths[k]] (features, PPI labels; any
 *                    width >= 1, no row alignment assumed)
 *   graph_tensors    host array of num_graph_tensors device pointers, fp32 [graph_rows[k], G] (QM9 targets)
 * A batch is the graphs order[start], ..., order[start + num_batch_graphs - 1] (order: int32 device array holding at least
 * start + num_batch_graphs entries, e.g. the epoch's permutation).  Outputs, caller-owned device buffers:
 *   out_node_tensors[k] [V, w_k], out_adjacency_lists[l] [E_l, 2] (node ids shifted by the graph's first node in the
 *   batch; batch-graph order, then the graph's own order), out_num_incoming [L, V], out_graph_nodes_list int32 [V] (batch
 *   index of every node's graph; may be NULL), out_graph_tensors[k] [graph_rows[k], num_batch_graphs].
 * The values are copies: the result is bit-identical to the host batcher's.  batch_nodes (V) and batch_edges (host [L],
 * E_l) are the caller's totals, known from host-side per-graph counts; the batch's offsets are computed on the device
 * (exclusive scans in the workspace).  Nothing is written past the caller's totals.  If a device total differs from the
 * caller's, or an order entry lies outside [0, G), the pack still completes without a fault, and `status` (int32 device
 * word, may be NULL) receives RGNN_PACK_* bits -- 0 when the batch is consistent; it is written on every call.
 * No allocation, no atomics, no synchronisation: capturable into a CUDA graph (a replay reads `order` as it is then).
 * Workspace: rgnn_pack_workspace_bytes(num_batch_graphs, L), 16-byte aligned (the contract stated above
 * rgnn_workspace_bytes).  Invalid arguments (negative counts, L outside [1, RGNN_MAX_EDGE_TYPES], more than
 * RGNN_PACK_MAX_TENSORS tensors of a kind, NULL required pointers) return RGNN_E_INVALID and a short workspace
 * RGNN_E_WORKSPACE, both before anything is enqueued.  The lists are ready for rgnn_plan_create_ex(...,
 * RGNN_PLAN_DEFERRED_CHECK) with V = batch_nodes; when the set's local ids were checked against their graphs' sizes once,
 * no per-batch check is needed. */
#define RGNN_PACK_MAX_TENSORS 8
#define RGNN_PACK_NODES_MISMATCH 1   /* the batch's node count differs from batch_nodes */
#define RGNN_PACK_EDGES_MISMATCH 2   /* some type's edge count differs from batch_edges[l] */
#define RGNN_PACK_BAD_ORDER 4        /* an order entry lies outside [0, G) (that graph is skipped) */
RGNN_API size_t rgnn_pack_workspace_bytes(int32_t num_batch_graphs, int32_t num_edge_types);
RGNN_API int rgnn_pack_minibatch(int64_t num_graphs, int64_t num_nodes, int32_t num_edge_types,
                        const int64_t* node_offsets, const int64_t* const* edge_offsets,
                        const int32_t* const* adjacency_lists, const float* num_incoming,
                        int32_t num_node_tensors, const float* const* node_tensors, const int32_t* node_widths,
                        int32_t num_graph_tensors, const float* const* graph_tensors, const int32_t* graph_rows,
                        const int32_t* order, int64_t start, int32_t num_batch_graphs, int32_t batch_nodes,
                        const int64_t* batch_edges, float* const* out_node_tensors, int32_t* const* out_adjacency_lists,
                        float* out_num_incoming, int32_t* out_graph_nodes_list, float* const* out_graph_tensors,
                        int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---- building blocks exported for tests / other hosts ---------------------------------------
 * utils/utils.py:23-33: aggregate `data` [M, d] (rows in the ORIGINAL type-major message order)
 * to [V, d] with the plan's segments -- the tf.unsorted_segment_<agg> call of rgcn.py:110. */
RGNN_API int rgnn_segment_aggregate(const rgnn_plan_t* plan, const float* data, int32_t d, int aggregation,
                           float* out, void* stream);
/* The edge stage on per-node transformed states: out[v,:] = agg over the incoming edges (u,v) of every type l of
 * s * table[u,l,:], table [V, L, d] row-major, s = 1/(num_incoming[l,v] + 1e-7) or 1 when num_incoming is NULL
 * (gnns/rgcn.py:84-112 and ggnn.py:76-90 with the per-type Dense applied per node first).  The backward gives
 * d_table[u,l,:] = sum over the outgoing edges (u,v) of type l of s * grad_out[v,:] / div(v) for sum / mean / sqrt_n
 * (RGNN_E_UNSUPPORTED for max); the reverse index is built inside the plan on first use. */
RGNN_API int rgnn_edge_aggregate_forward(const rgnn_plan_t* plan, const float* table, int32_t d, const float* num_incoming,
                                int aggregation, float* out, void* stream);
RGNN_API int rgnn_edge_aggregate_backward(const rgnn_plan_t* plan, const float* grad_out, int32_t d,
                                 const float* num_incoming, int aggregation, float* d_table, void* stream);
/* C[M,N] = act(A[M,K] . B[K,N] + bias) on the tensor cores with 3xTF32 split accumulation
 * (fp32-accurate); the node-level Dense of every layer (A.1). bias may be NULL.  workspace: caller scratch of at least
 * rgnn_dense_workspace_bytes(m, k, n) bytes (weight images; split-K partial tiles of the backward) -- the library
 * allocates nothing per call. */
RGNN_API size_t rgnn_dense_workspace_bytes(int32_t m, int32_t k, int32_t n);
RGNN_API int rgnn_dense_forward(const float* a, int32_t m, int32_t k, const float* b, int32_t n,
                       const float* bias, int activation, float* c, void* workspace, size_t workspace_bytes, void* stream);
/* Gradients of the linear map C = A . B: grad_a [M,K] = grad_c . B^T, grad_b [K,N] = A^T . grad_c (split-K on the tensor
 * cores, deterministic).  Either output may be NULL.  The reference gets these from TF autodiff of its Dense kernels
 * (models/sparse_graph_model.py:253-260). */
RGNN_API int rgnn_dense_backward(const float* a, int32_t m, int32_t k, const float* b, int32_t n, const float* grad_c,
                        float* grad_a, float* grad_b, void* workspace, size_t workspace_bytes, void* stream);
/* tf.contrib.layers.layer_norm over the last axis, eps 1e-12 (A.5). */
RGNN_API int rgnn_layer_norm(const float* x, int32_t rows, int32_t d, const float* gamma, const float* beta,
                    float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RGNN_H_ */
