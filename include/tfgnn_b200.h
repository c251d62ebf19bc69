/*
 * tfgnn_b200.h — C ABI of the H100-native tf2_gnn message-passing hot path.
 *
 * The reference (microsoft/tf2-gnn) is pure Python on TensorFlow: it has no FFI of its own.
 * Each entry point below replaces a span of reference Python that runs once per layer (or once
 * per batch) inside tf2_gnn.layers.GNN._internal_call; the span is cited next to it
 * (paths relative to /root/reference/).  INTEGRATION.md shows the ctypes stub a maintainer
 * adds on the reference side.
 *
 * Conventions
 *   - Every data pointer is a DEVICE pointer (zero-copy from DLPack / tensor.data_ptr()).
 *     The only host pointers are the small arrays of per-edge-type pointers / sizes, which
 *     are read during the call and may be freed right after it returns.
 *   - float32 node states / weights, int32 adjacency: [E,2] row-major [src,tgt] pairs
 *     (message_passing.py:102-104,195-196; gnn.py:222-228).
 *   - The caller owns all inputs, weights and the PRE-ALLOCATED output.  The library owns only
 *     the opaque tfgnn_batch_t (its CSR), released by tfgnn_b200_free_batch.
 *   - The output of a layer call must not overlap its node-state input (every target gathers arbitrary
 *     source rows); entries that work in place say so.
 *   - All work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = legacy default
 *     stream).  No entry point synchronises the device except tfgnn_b200_prepare with
 *     TFGNN_PREPARE_VALIDATE and tfgnn_b200_free_batch.
 *   - Return value 0 = success; otherwise a TFGNN_ERR_* code and tfgnn_b200_last_error()
 *     (thread-local) describes it.  There is NO CPU fallback anywhere in this library.
 */
#ifndef TFGNN_B200_H_
#define TFGNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFGNN_B200_ABI_VERSION 1
/* The library is built with -fvisibility=hidden: only the entry points declared here are exported. */
#if defined(__GNUC__)
#define TFGNN_API __attribute__((visibility("default")))
#else
#define TFGNN_API
#endif
#define TFGNN_MAX_EDGE_TYPES 32
#define TFGNN_MAX_PEERS 15 /* peer replicas of tfgnn_b200_rgcn_fwd_allgather (one NVSwitch domain: <= 16 GPUs) */

typedef struct tfgnn_batch tfgnn_batch_t;

enum {
  TFGNN_OK = 0,
  TFGNN_ERR_INVALID_ARGUMENT = 1, /* maps to Python ValueError  */
  TFGNN_ERR_CUDA = 2,             /* maps to Python RuntimeError */
  TFGNN_ERR_UNSUPPORTED = 3,      /* maps to Python NotImplementedError (never a fallback) */
  TFGNN_ERR_INDEX_OUT_OF_RANGE = 4 /* maps to Python IndexError (TF-CPU raises on bad ids) */
};

/* tf2_gnn/utils/param_helpers.py:7-19 */
enum { TFGNN_AGG_SUM = 0, TFGNN_AGG_MEAN = 1, TFGNN_AGG_MAX = 2, TFGNN_AGG_SQRT_N = 3 };
/* tf2_gnn/utils/param_helpers.py:22-42 ; activation.py:7-14 */
enum {
  TFGNN_ACT_NONE = 0, TFGNN_ACT_RELU = 1, TFGNN_ACT_TANH = 2, TFGNN_ACT_LEAKY_RELU = 3,
  TFGNN_ACT_ELU = 4, TFGNN_ACT_SELU = 5, TFGNN_ACT_GELU = 6,
  TFGNN_ACT_SIGMOID = 7 /* not in the reference's name table: tf.nn.sigmoid of the readout weights,
                           nodes_to_graph_representation.py:174-175 */
};
/* layer flags */
enum {
  TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING = 1u << 0, /* gnn_edge_mlp.py:102-106 */
  TFGNN_FLAG_ACT_BEFORE_AGGREGATION = 1u << 1,    /* message_passing.py:169-177 */
  TFGNN_FLAG_USE_TARGET_STATE = 1u << 2           /* gnn_edge_mlp.py:93-98 */
};
/* execution path (SURVEY.md §8b) */
enum {
  TFGNN_PATH_AUTO = 0,
  TFGNN_PATH_ATOMIC = 1,     /* per-edge red.global.add, no CSR use (evidence path)      */
  TFGNN_PATH_SORTED = 2,     /* CSR segmented reduce + fp32 SIMT node-level GEMM         */
  TFGNN_PATH_SORTED_TC = 3,  /* CSR segmented reduce + 3xTF32 wgmma node-level GEMM       */
  TFGNN_PATH_FUSED_TC = 4    /* one kernel: gather-reduce -> wgmma -> activation         */
};
enum {
  TFGNN_PREPARE_VALIDATE = 1u << 0,
  TFGNN_PREPARE_TRANSPOSE = 1u << 1, /* key the CSR by SOURCE: the edge list of the backward pass (messages flow tgt->src) */
  /* Backward CSR of a target-range shard (tfgnn_b200_prepare_sharded only; takes precedence over TFGNN_PREPARE_TRANSPOSE):
   * keeps the edges whose TARGET lies in [target_begin, target_begin + target_count), keys them by (type, global source)
   * over all num_nodes_total sources (row_ptr has L*num_nodes_total+1 entries) and stores the LOCAL target id
   * tgt - target_begin, ascending within each segment.  With target_begin = 0, target_count = num_nodes_total it is the
   * TFGNN_PREPARE_TRANSPOSE batch. */
  TFGNN_PREPARE_TRANSPOSE_OWNED = 1u << 2
};

TFGNN_API int tfgnn_b200_abi_version(void);
TFGNN_API const char* tfgnn_b200_last_error(void);

/* Per-batch preprocessing, reused by every layer of the stack (the adjacency is layer-invariant:
 * gnn.py:278,301).  Builds, per edge type, the edges sorted by target (CSR keyed by
 * type*V + target) and with it the in-degree table that the reference recomputes every layer in
 * calculate_type_to_num_incoming_edges (message_passing.py:190,230-263).
 *   adj        host array of L device pointers, adj[l] = int32[num_edges[l], 2]
 *   num_edges  host array of L edge counts (may be 0: graph_dataset.py:244)
 * Edges whose src or tgt lies outside [0,V) are dropped; with TFGNN_PREPARE_VALIDATE the call
 * synchronises the stream and returns TFGNN_ERR_INDEX_OUT_OF_RANGE instead. */
TFGNN_API int tfgnn_b200_prepare(const int32_t* const* adj, const int64_t* num_edges, int32_t num_edge_types,
                       int64_t num_nodes, uint32_t prepare_flags, tfgnn_batch_t** out_batch,
                       void* stream);
/* Target-range shard of ONE graph too large for a GPU (SURVEY.md §8e): this batch owns the targets
 * [target_begin, target_begin+target_count) of a graph with num_nodes_total nodes.  adj may hold the
 * whole edge list (edges into other shards are skipped) or a pre-filtered one; ids stay GLOBAL.
 * Layer calls on such a batch take the full source table h[num_nodes_total, D] (all-gathered over the
 * ranks once per layer) and write out[target_count, H]; target-side reads use rows target_begin+v. */
TFGNN_API int tfgnn_b200_prepare_sharded(const int32_t* const* adj, const int64_t* num_edges,
                               int32_t num_edge_types, int64_t num_nodes_total, int64_t target_begin,
                               int64_t target_count, uint32_t prepare_flags, tfgnn_batch_t** out_batch,
                               void* stream);
TFGNN_API int tfgnn_b200_free_batch(tfgnn_batch_t* batch);

/* Introspection of the opaque batch (device pointers stay owned by the batch):
 * row_ptr int32[L*V+1], src_sorted int32[num_valid_edges]. */
TFGNN_API int tfgnn_b200_batch_info(const tfgnn_batch_t* batch, int64_t* num_nodes, int32_t* num_edge_types,
                          int64_t* num_edges_total, const int32_t** row_ptr,
                          const int32_t** src_sorted);

/* Copy the CSR into caller-owned device buffers (row_ptr_out int32[L*V+1], src_sorted_out
 * int32[num_edges_total]); either may be NULL. */
TFGNN_API int tfgnn_b200_batch_export_csr(const tfgnn_batch_t* batch, int32_t* row_ptr_out,
                                int32_t* src_sorted_out, void* stream);

/* calculate_type_to_num_incoming_edges (message_passing.py:230-263): out = float32[L, V]. */
TFGNN_API int tfgnn_b200_in_degree(const tfgnn_batch_t* batch, float* out, void* stream);

/* GNN_Edge_MLP / RGCN forward (gnn_edge_mlp.py:84-107 + message_passing.py:95-218):
 *   out[v] = agg_{l, (u,v) in A_l} [ MLP_l(h_u [|| h_v]) / (c_{v,l}+1e-7) ]   with activation before
 *   or after the aggregation.  RGCN = num_hidden_layers 0, no target state, normalise (rgcn.py:50-59).
 *   mlp_weights  host array of L*(num_hidden_layers+1) device pointers, type-major; layer 0 is
 *                [D_in, H] with D_in = D or 2D (rows [0,D) act on h_src, [D,2D) on h_tgt),
 *                further layers [H, H]; no biases (test_RGCN.py:35-39).
 *   h [V, D], out [V, H]. */
TFGNN_API int tfgnn_b200_edge_mlp_fwd(tfgnn_batch_t* batch, const float* h, int32_t D,
                            const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H,
                            uint32_t flags, int32_t aggregation, int32_t activation, int32_t path,
                            float* out, void* stream);

/* Backward of tfgnn_b200_edge_mlp_fwd with ONE hidden layer (the class defaults of GNN_Edge_MLP and RGIN; the reference
 * differentiates with tf.GradientTape, models/graph_task_model.py:338-365) in the hoisted form of the forward: no tensor has
 * a per-edge dimension.  batch_t is the SAME adjacency prepared with TFGNN_PREPARE_TRANSPOSE.  mlp_weights = the L*2 tables
 * of the forward (U_l [D_in, H], W2_l [H, H], type-major); out = saved forward output, grad_out = dL/dout [V,H]; writes
 * grad_h [V,D] (may be NULL) and grad_weights, the L*2 gradients in the same order.  The hidden ReLU's derivative is
 * [pre-activation > 0] (0 at 0, as TF's ReluGrad).
 * Supported: num_hidden_layers 1, sum/mean/sqrt_n aggregation, activation after aggregation, every activation (gelu
 * through a recomputed pre-activation), source-only or source+target state input (TFGNN_FLAG_USE_TARGET_STATE), D and H
 * multiples of 4, H <= 512.  Anything else returns TFGNN_ERR_UNSUPPORTED (0 hidden layers: tfgnn_b200_rgcn_bwd).
 * On a target-range shard (batch from tfgnn_b200_prepare_sharded over targets [lo, hi)), batch_t must be the same
 * adjacency and range prepared with TFGNN_PREPARE_TRANSPOSE_OWNED.  h is then the full [num_nodes_total, D] table, out and
 * grad_out have hi-lo rows, and the call writes THIS SHARD'S CONTRIBUTION: grad_h [num_nodes_total, D] (every row; the
 * target-state terms land on rows [lo, hi)) and every weight gradient.  The contributions of all shards sum to the
 * unsharded gradients.  Each shard's result is run-to-run reproducible (no atomics).  An empty shard, or a batch without
 * edge types, writes zeros. */
TFGNN_API int tfgnn_b200_edge_mlp_bwd(tfgnn_batch_t* batch, tfgnn_batch_t* batch_t, const float* h, int32_t D,
                            const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H, uint32_t flags,
                            int32_t aggregation, int32_t activation, const float* out, const float* grad_out,
                            float* grad_h, float* const* grad_weights, void* stream);

/* RGCN convenience entry (rgcn.py:12-62): edge_mlp_fwd with 0 hidden layers, source state only. */
TFGNN_API int tfgnn_b200_rgcn_fwd(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W,
                        int32_t H, uint32_t flags, int32_t aggregation, int32_t activation,
                        int32_t path, float* out, void* stream);

/* RGCN layer followed by LayerNormalization (gnn.py:299-321 with use_inter_layer_layernorm, e.g. QM9_RGCN.json): when the
 * layer takes the fused kernel with one N pass (H <= 64) the normalisation runs in the kernel's epilogue - each row's
 * accumulators sit in the registers of one lane quad, so mean / variance are two shuffle reductions and the [V,H] round trip
 * through HBM of a separate LayerNorm pass disappears.  Otherwise the stand-alone kernel is applied in place: the result is
 * the same either way.  out = LayerNorm(rgcn(h)); the un-normalised layer output is not produced. */
TFGNN_API int tfgnn_b200_rgcn_ln_fwd(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W, int32_t H,
                                     uint32_t flags, int32_t aggregation, int32_t activation, int32_t path,
                                     const float* ln_gamma, const float* ln_beta, float ln_epsilon, float* out, void* stream);

/* Layer + all-gather in ONE kernel over peer memory (SURVEY.md §8e case 2: one graph partitioned by target range over the
 * GPUs of an NVSwitch domain, tfgnn_b200_prepare_sharded).  Same computation as tfgnn_b200_rgcn_fwd on the shard, but the
 * epilogue of the fused kernel stores every finished 128-row output tile into the caller's own table AND into the peers'
 * copies of it: out_replicas[r] is rank r's [num_nodes_total, H] node-state table as mapped into THIS process (CUDA P2P over
 * NVLink: a symmetric-memory allocator, cudaIpcOpenMemHandle, NVSHMEM ...; out_replicas[own_rank] is local memory), rows
 * target_begin + v.  When every rank has run the call, each replica holds the all-gathered new node states: the per-layer
 * all-gather of the reference-sized alternative (ncclAllGather after the layer) overlaps the layer tile by tile instead of
 * following it.  out_multicast (may be NULL): a MULTICAST mapping of the same tables (NVSwitch multicast object, e.g.
 * cuMulticastBindMem / a symmetric-memory multicast pointer): the epilogue then issues ONE multimem.st per 16 bytes and the
 * switch replicates it to every GPU, so a rank's NVLink egress per layer is its own rows once instead of once per peer.
 * The caller double-buffers the tables across layers (layer k reads table k%2, writes table (k+1)%2) and
 * synchronises the ranks between layers (a few-microsecond signal exchange).
 * TFGNN_ERR_UNSUPPORTED when the shard does not take the fused kernel (D % 32, H % 16, H <= 512, linear messages,
 * sum/mean/sqrt_n, activation after aggregation): fall back to the layer call + an all-gather. */
TFGNN_API int tfgnn_b200_rgcn_fwd_allgather(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W, int32_t H,
                                            uint32_t flags, int32_t aggregation, int32_t activation,
                                            float* const* out_replicas, int32_t num_replicas, int32_t own_rank,
                                            float* out_multicast, void* stream);

/* Backward of tfgnn_b200_rgcn_fwd (SURVEY.md §8f-1; the reference differentiates with tf.GradientTape,
 * models/graph_task_model.py:338-365).  batch_t is the SAME adjacency prepared with TFGNN_PREPARE_TRANSPOSE.
 * out = saved forward output, grad_out = dL/dout [V,H]; writes grad_h [V,D] (may be NULL) and grad_W[l] [D,H].
 * Supported: sum/mean/sqrt_n aggregation, activation after aggregation, activations none/relu/tanh/leaky_relu/
 * elu/selu (derivative from the output) and gelu (pre-activation recomputed), source-only or source+target state input (W[l] = [D,H] or [2D,H],
 * TFGNN_FLAG_USE_TARGET_STATE); D and H multiples of 4.
 * On a target-range shard (batch from tfgnn_b200_prepare_sharded over targets [lo, hi)), batch_t must be the same
 * adjacency and range prepared with TFGNN_PREPARE_TRANSPOSE_OWNED.  h is then the full [num_nodes_total, D] table, out and
 * grad_out have hi-lo rows, and the call writes THIS SHARD'S CONTRIBUTION: grad_h [num_nodes_total, D] (every row; rows no
 * owned edge reads are zero; the target-state term lands on rows [lo, hi)) and grad_W[l].  The contributions of all shards
 * sum to the unsharded gradients (a reduce-scatter of grad_h and an all-reduce of grad_W across the ranks).  Each shard's
 * result is run-to-run reproducible (no atomics).  An empty shard writes zeros. */
TFGNN_API int tfgnn_b200_rgcn_bwd(tfgnn_batch_t* batch, tfgnn_batch_t* batch_t, const float* h, int32_t D,
                        const float* const* W, int32_t H, uint32_t flags, int32_t aggregation,
                        int32_t activation, const float* out, const float* grad_out, float* grad_h,
                        float* const* grad_W, void* stream);

/* GGNN (ggnn.py:68-89): edge-MLP messages (class default: 0 hidden layers, source state only,
 * normalised), aggregation, NO message activation, then Keras GRUCell(units=H, reset_after=True):
 * gru_kernel [H,3H] acts on the aggregated messages, gru_recurrent_kernel [H,3H] on the state h
 * (D == H required, ggnn.py:30), gru_bias [2,3H]; gate order z,r,h. */
TFGNN_API int tfgnn_b200_ggnn_fwd(tfgnn_batch_t* batch, const float* h, int32_t D,
                        const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H,
                        uint32_t flags, int32_t aggregation, const float* gru_kernel,
                        const float* gru_recurrent_kernel, const float* gru_bias, int32_t path,
                        float* out, void* stream);

/* Backward of tfgnn_b200_ggnn_fwd (SURVEY.md section 8f-1; the reference differentiates through GGNN with
 * tf.GradientTape, models/graph_task_model.py:338-365).  Recomputes the forward intermediates from h; batch_t is
 * the TFGNN_PREPARE_TRANSPOSE batch of the same adjacency lists.  Writes grad_h [V,H], grad_W[l] [H,H],
 * grad_gru_kernel [H,3H], grad_gru_recurrent_kernel [H,3H], grad_gru_bias [2,3H].
 * Supported: 0 hidden layers in the message MLPs, source state only, sum / mean / sqrt_n aggregation, H % 4 == 0.
 * On a target-range shard the pair (batch, batch_t) is as for tfgnn_b200_rgcn_bwd: h is the full [num_nodes_total, H]
 * table, grad_out has hi-lo rows, the GRU reads its state from rows [lo, hi) of h, and the call writes this shard's
 * contribution to grad_h [num_nodes_total, H] (GRU direct and recurrent terms on rows [lo, hi)), to grad_W and to the GRU
 * gradients; the contributions of all shards sum to the unsharded gradients.  An empty shard writes zeros. */
TFGNN_API int tfgnn_b200_ggnn_bwd(tfgnn_batch_t* batch, tfgnn_batch_t* batch_t, const float* h, int32_t D,
                        const float* const* W, int32_t H, uint32_t flags, int32_t aggregation,
                        const float* gru_kernel, const float* gru_recurrent_kernel, const float* gru_bias,
                        const float* grad_out, float* grad_h, float* const* grad_W, float* grad_gru_kernel,
                        float* grad_gru_recurrent_kernel, float* grad_gru_bias, void* stream);

/* RGIN (rgin.py:88-106): edge MLP messages, aggregation, optional aggregation MLP
 * (aggr_weights: host array of num_aggr_layers device pointers [H,H], may be NULL/0), activation. */
TFGNN_API int tfgnn_b200_rgin_fwd(tfgnn_batch_t* batch, const float* h, int32_t D,
                        const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H,
                        uint32_t flags, int32_t aggregation, int32_t activation,
                        const float* const* aggr_weights, int32_t num_aggr_layers, int32_t path,
                        float* out, void* stream);

/* GNN-FiLM (gnn_film.py:83-108): m = gamma_l(h_v) * EdgeMLP_l(...) + beta_l(h_v),
 * [gamma|beta] = h_v F_l, film_weights: host array of L device pointers [D, 2H] (no hidden layers). */
TFGNN_API int tfgnn_b200_film_fwd(tfgnn_batch_t* batch, const float* h, int32_t D,
                        const float* const* mlp_weights, int32_t num_hidden_layers,
                        const float* const* film_weights, int32_t H, uint32_t flags,
                        int32_t aggregation, int32_t activation, int32_t path, float* out,
                        void* stream);

/* Backward of tfgnn_b200_film_fwd (the reference differentiates with tf.GradientTape,
 * models/graph_task_model.py:338-365) in the aggregate-then-transform form: no tensor has a per-edge dimension.
 * batch_t is the SAME adjacency prepared with TFGNN_PREPARE_TRANSPOSE.  out = saved forward output, grad_out = dL/dout
 * [V,H]; writes grad_h [V,D] (may be NULL), grad_W[l] [D,H] or [2D,H] (the edge-MLP kernels, mlp_weights) and grad_film[l]
 * [D,2H] (the FiLM kernels, film_weights).
 * Supported: 0 hidden layers in the edge MLPs and in the FiLM MLPs, sum/mean/sqrt_n aggregation, activation after
 * aggregation, activations none/relu/tanh/leaky_relu/elu/selu (derivative from the output) and gelu (pre-activation
 * recomputed), source-only or source+target state input (TFGNN_FLAG_USE_TARGET_STATE); D and H multiples of 4.  Anything
 * else returns TFGNN_ERR_UNSUPPORTED.
 * On a target-range shard (batch from tfgnn_b200_prepare_sharded over targets [lo, hi)), batch_t must be the same
 * adjacency and range prepared with TFGNN_PREPARE_TRANSPOSE_OWNED.  h is then the full [num_nodes_total, D] table, out and
 * grad_out have hi-lo rows, and the call writes THIS SHARD'S CONTRIBUTION: grad_h [num_nodes_total, D] (every row; the
 * FiLM and target-state terms land on rows [lo, hi)), grad_W[l] and grad_film[l].  The contributions of all shards sum to
 * the unsharded gradients.  Each shard's result is run-to-run reproducible (no atomics).  An empty shard, or a batch
 * without edge types, writes zeros. */
TFGNN_API int tfgnn_b200_film_bwd(tfgnn_batch_t* batch, tfgnn_batch_t* batch_t, const float* h, int32_t D,
                        const float* const* mlp_weights, const float* const* film_weights, int32_t H,
                        uint32_t flags, int32_t aggregation, int32_t activation, const float* out,
                        const float* grad_out, float* grad_h, float* const* grad_W, float* const* grad_film,
                        void* stream);

/* RGAT (rgat.py:91-163): per-type projection W_l [D,H], attention a_l [K, 2H/K]; softmax over all
 * incoming edges of all types jointly, per head; activation after. */
TFGNN_API int tfgnn_b200_rgat_fwd(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W,
                        const float* const* attention, int32_t H, int32_t num_heads,
                        int32_t activation, int32_t path, float* out, void* stream);

/* Backward of tfgnn_b200_rgat_fwd (the reference differentiates with tf.GradientTape,
 * models/graph_task_model.py:338-365) without per-edge tensors: every temporary is node-sized.  batch_t is the SAME adjacency
 * prepared with TFGNN_PREPARE_TRANSPOSE.  path = the forward's path: P = h W_l and the score halves are recomputed with the
 * forward's bits.  out = saved forward output, grad_out = dL/dout [V,H]; writes grad_h [V,D] (may be NULL), grad_W[l] [D,H]
 * and grad_attention[l] [K, 2H/K].
 * Supported: D % 4 == 0, (H / num_heads) % 4 == 0, H <= 512, activations none/relu/tanh/leaky_relu/elu/selu (derivative
 * from the output) and gelu (pre-activation recomputed).  Anything else (and TFGNN_PATH_ATOMIC) returns
 * TFGNN_ERR_UNSUPPORTED.
 * On a target-range shard (batch from tfgnn_b200_prepare_sharded over targets [lo, hi)), batch_t must be the same
 * adjacency and range prepared with TFGNN_PREPARE_TRANSPOSE_OWNED.  h is then the full [num_nodes_total, D] table, out and
 * grad_out have hi-lo rows, and the call writes THIS SHARD'S CONTRIBUTION: grad_h [num_nodes_total, D] (every row),
 * grad_W[l] and grad_attention[l].  The contributions of all shards sum to the unsharded gradients.  An empty shard, or a
 * batch without edge types, writes zeros.
 * No float atomics: hub targets (more than 2048 incoming edges) are cut into fixed chunks whose partials are combined in
 * chunk order, so every call, and each shard's contribution, is bitwise reproducible for the same inputs. */
TFGNN_API int tfgnn_b200_rgat_bwd(tfgnn_batch_t* batch, tfgnn_batch_t* batch_t, const float* h, int32_t D,
                        const float* const* W, const float* const* attention, int32_t H, int32_t num_heads,
                        int32_t activation, int32_t path, const float* out, const float* grad_out, float* grad_h,
                        float* const* grad_W, float* const* grad_attention, void* stream);

/* Node-level dense layer out = act(x W), x [V,K], W [K,N], no bias — the op behind every
 * tf.keras.layers.Dense(use_bias=False) on the path (gnn.py:136-141,165-169) and the building
 * block of the fp32-accurate node-level contractions.  path: 0 auto, 2 SIMT fp32, 3 wgmma 3xTF32. */
TFGNN_API int tfgnn_b200_dense_fwd(const float* x, const float* W, float* out, int64_t V, int32_t K, int32_t N,
                         int32_t activation, int32_t path, void* stream);

/* The three stock ops of the reference's generic MessagePassing.call, for user-defined
 * _message_function plugins (message_passing.py:64-93) and the literal per-edge path:
 *   gather_rows               tf.nn.embedding_lookup            message_passing.py:197-206
 *   unsorted_segment_reduce   tf.math.unsorted_segment_{sum,mean,max,sqrt_n}  :172-174
 *   activation                get_activation_function(...)      :169-177
 * ids / segment_ids are int32 with an element stride (2 addresses a column of an [E,2] list). */
TFGNN_API int tfgnn_b200_gather_rows(const float* table, int64_t num_rows, int32_t D, const int32_t* ids,
                           int64_t ids_stride, int64_t n, float* out, void* stream);
TFGNN_API int tfgnn_b200_unsorted_segment_reduce(const float* data, const int32_t* segment_ids,
                                       int64_t ids_stride, int64_t M, int32_t H,
                                       int64_t num_segments, int32_t aggregation, float* out,
                                       void* stream);
TFGNN_API int tfgnn_b200_activation(const float* x, int64_t n, int32_t activation, float* out, void* stream);

/* Node-level glue of GNN._internal_call around the message-passing layers (gnn.py:291-296,317-321):
 *   residual_average   out = (x + last) / 2                      gnn.py:294-295
 *   layer_norm         tf.keras.layers.LayerNormalization(axis=-1, epsilon) over each row  gnn.py:318-321
 * x, last, out: [V, H] contiguous; gamma, beta: [H]. */
TFGNN_API int tfgnn_b200_residual_average(const float* x, const float* last, float* out, int64_t n, void* stream);
TFGNN_API int tfgnn_b200_layer_norm(const float* x, const float* gamma, const float* beta, int64_t V, int32_t H,
                          float epsilon, float* out, void* stream);

/* ---- Training-time node-level glue (SURVEY.md section 8f-1/3; the reference differentiates gnn.py:279-327 with
 * tf.GradientTape, models/graph_task_model.py:338-365) -------------------------------------------------------------
 *   dense_bwd        backward of out = act(x W + bias): grad_x [V,K] (or NULL), grad_W [K,N] (or NULL), grad_bias [N] (or
 *                    NULL); `out` is the saved forward output (gelu recomputes the pre-activation)
 *   layer_norm_bwd   backward of tfgnn_b200_layer_norm: grad_x (or NULL), grad_gamma, grad_beta (fixed-order column sums)
 *   dropout          tf.nn.dropout(x, rate): out = x * mask / (1 - rate), mask ~ Bernoulli(1 - rate) from Philox4x32-10
 *                    keyed by (seed, offset + element index / 4).  Deterministic per (seed, offset); the backward pass is
 *                    the same call on the incoming gradient.  (TensorFlow's own stream cannot be reproduced: parity of
 *                    training-time dropout is distributional.)
 *   axpby            out = alpha * a + beta * b (b NULL: alpha * a): residual average and its backward */
TFGNN_API int tfgnn_b200_dense_bwd(const float* x, const float* W, const float* bias, const float* out, const float* grad_out,
                                   int64_t V, int32_t K, int32_t N, int32_t activation, float* grad_x, float* grad_W,
                                   float* grad_bias, void* stream);
TFGNN_API int tfgnn_b200_layer_norm_bwd(const float* x, const float* gamma, const float* grad_out, int64_t V, int32_t H,
                                        float epsilon, float* grad_x, float* grad_gamma, float* grad_beta, void* stream);
TFGNN_API int tfgnn_b200_dropout(const float* x, int64_t n, float rate, uint64_t seed, uint64_t offset, float* out,
                                 void* stream);
TFGNN_API int tfgnn_b200_axpby(const float* a, float alpha, const float* b, float beta, int64_t n, float* out, void* stream);

/* ---- Differentiable generic path (SURVEY.md section 8f-1) -----------------------------------------------------------
 * The reference trains every variant by differentiating its literal op sequence (message_passing.py:95-218) with
 * tf.GradientTape.  Variants without a fused backward kernel train through the same sequence here; these are the
 * remaining forward / backward ops of that sequence (gather_rows <-> unsorted_segment_reduce(sum) are each other's
 * backward, dense_bwd is above):
 *   activation_bwd     grad_in = grad_out * act'(.); `ref` = forward OUTPUT (gelu: forward INPUT)
 *   row_scale          out[m,:] = x[m,:] * f(s[m]); f = s | 1/(s+1e-7) | 1/max(s,1) | 1/sqrt(max(s,1))   (modes 0..3)
 *   mul_add            out = a * b (+ c) on 2-D views with leading dimensions (FiLM: gamma * m + beta, gnn_film.py:105-107)
 *   segment_max_bwd    gradient of unsorted_segment_max: to the elements that attain the maximum, shared among ties
 *   softmax_apply      exp(s - m) or exp((s - m) - log z) on per-element gathered segment max / sum (the two elementwise
 *                      stages of dpu_utils unsorted_segment_(log_)softmax: rgat.py:147-151,
 *                      nodes_to_graph_representation.py:179-185)
 *   head_scale         out[e, k*d+i] = w[e,k] * x[e, k*d+i]  (attention-weighted messages rgat.py:152-155, readout :219-220)
 *   head_dot           out[e,k] = sum_i a[e,k*d+i] * b[e,k*d+i]  (gradient of head_scale with respect to w)
 *   gru_gate_bwd       backward of gru_gate_fwd: grad_gx, grad_gh [V,3H] and the direct path grad_out * z [V,H] */
TFGNN_API int tfgnn_b200_activation_bwd(const float* ref, const float* grad_out, int64_t n, int32_t activation,
                                        float* grad_in, void* stream);
TFGNN_API int tfgnn_b200_row_scale(const float* x, const float* s, int64_t M, int32_t H, int32_t mode, float* out,
                                   void* stream);
TFGNN_API int tfgnn_b200_mul_add(const float* a, int32_t lda, const float* b, int32_t ldb, const float* c, int32_t ldc,
                                 int64_t M, int32_t H, float* out, int32_t ldo, void* stream);
TFGNN_API int tfgnn_b200_segment_max_bwd(const float* data, const int32_t* segment_ids, int64_t ids_stride,
                                         const float* segment_out, const float* segment_grad, int64_t M, int32_t H,
                                         int64_t num_segments, float* grad_data, void* stream);
TFGNN_API int tfgnn_b200_softmax_apply(const float* scores, const float* seg_max_per_elem, const float* seg_sum_per_elem,
                                       int64_t n, float* out, void* stream);
TFGNN_API int tfgnn_b200_head_scale(const float* x, const float* w, int64_t M, int32_t num_heads, int32_t head_dim, float* out,
                                    void* stream);
TFGNN_API int tfgnn_b200_head_dot(const float* a, const float* b, int64_t M, int32_t num_heads, int32_t head_dim, float* out,
                                  void* stream);
TFGNN_API int tfgnn_b200_gru_gate_bwd(const float* gx, const float* gh, const float* h, const float* grad_out, int64_t num_rows,
                                      int32_t H, float* grad_gx, float* grad_gh, float* grad_h_direct, void* stream);

/* ---- Graph-level readout and global exchange (SURVEY.md section 8f-4) ---------------------------------------------
 * Segment primitives keyed by node_to_graph_map, which is non-decreasing (graph_dataset.py:211-217; the reference's own
 * tf.math.segment_sum requires it), so a graph is the contiguous row range graph_ptr[g] .. graph_ptr[g+1].
 *   graph_offsets          node_to_graph_map int32[V] -> graph_ptr int32[G+1]; validate != 0 synchronises the stream and
 *                          returns TFGNN_ERR_INVALID_ARGUMENT for ids that decrease or fall outside [0, G)
 *   segment_softmax        scores [V,K] -> weights [V,K]: per (graph, head) exp((s - max) - log(sum exp(s - max)))
 *                          = dpu_utils unsorted_segment_softmax          nodes_to_graph_representation.py:176-186
 *   weighted_segment_sum   out[g, k*d+c] = sum_{v in g} weights[v,k] * node_reprs[v, k*d+c], d = repr_dim/num_heads
 *                          (weights NULL: plain tf.math.segment_sum; mean != 0: segment_mean)      :204-227
 *   gathered_add           out[v,:] = act((a[v,:] + b[index[v],:]) * scale); index NULL = identity
 *                          (mean exchange (x + g[n2g]) / 2, graph_global_exchange.py:124; hidden layer of the MLP exchange)
 *   gru_gate_fwd           Keras GRUCell(reset_after=True) gate math on precomputed gx = inputs K + b0 (rows picked by
 *                          gx_row_index, NULL = identity) and gh = h U + b1        graph_global_exchange.py:147-152
 *   clamp                  in-place transformation_mlp_result_{lower,upper}_bound   nodes_to_graph_representation.py:194-197
 *   dense_bias_fwd         out = act(x W + bias) (bias [N] or NULL)                 MLPs with use_biases, GRU halves */
TFGNN_API int tfgnn_b200_graph_offsets(const int32_t* node_to_graph_map, int64_t num_nodes, int32_t num_graphs,
                                       int32_t* graph_ptr, int32_t validate, void* stream);
TFGNN_API int tfgnn_b200_segment_softmax(const float* scores, const int32_t* graph_ptr, int32_t num_graphs,
                                         int32_t num_heads, float* out, void* stream);
TFGNN_API int tfgnn_b200_weighted_segment_sum(const float* node_reprs, const float* weights, const int32_t* graph_ptr,
                                              int32_t num_graphs, int32_t repr_dim, int32_t num_heads, int32_t mean,
                                              float* out, void* stream);
TFGNN_API int tfgnn_b200_gathered_add(const float* a, const float* b, const int32_t* index, int64_t num_rows, int32_t H,
                                      float scale, int32_t activation, float* out, void* stream);
TFGNN_API int tfgnn_b200_gru_gate_fwd(const float* gx, const int32_t* gx_row_index, const float* gh, const float* h,
                                      int64_t num_rows, int32_t H, float* out, void* stream);
TFGNN_API int tfgnn_b200_clamp(float* x, int64_t n, float lower, float upper, int32_t has_lower, int32_t has_upper,
                               void* stream);
TFGNN_API int tfgnn_b200_dense_bias_fwd(const float* x, const float* W, const float* bias, float* out, int64_t V, int32_t K,
                                        int32_t N, int32_t activation, int32_t path, void* stream);

/* Backward of the readout and the exchange combines on the same row ranges.  No float atomics: every result is a function
 * of its inputs alone (bitwise equal run to run, independent of the launch geometry).
 *   segment_sum_rows       out[g,:] = sum of data[v,:] over graph_ptr[g] <= v < graph_ptr[g+1] (zeros for an empty graph): the
 *                          adjoint of table[node_to_graph_map].  Rows are reduced in row order inside fixed 64-row chunks
 *                          and a graph's chunk sums are added in a fixed order, so few long graphs and many short ones
 *                          both fill the device
 *   readout_bwd            backward of weighted_segment_sum through the weighting (tfgnn_readout_mode_t) and the clamp.
 *                          node_reprs [V,GD] is the transformation result BEFORE the clamp, weights [V,K] the forward's
 *                          softmax / sigmoid output (NULL for none / average), out [G,GD] the forward result (softmax only).
 *                          With g = node_to_graph_map[v], R = clamp(node_reprs), d = GD/K:
 *                            grad_reprs[v,kd+c] = w[v,k] grad_out[g,kd+c]  (none: w = 1, average: 1/max(n_g,1)); zero where the
 *                              clamp cut: tf.maximum / tf.minimum pass the gradient where x >= lower resp. x <= upper
 *                            dw[v,k] = sum_c grad_out[g,kd+c] R[v,kd+c]
 *                            grad_scores[v,k] = dw w (1 - w)  (sigmoid)  |  w (dw - sum_c grad_out[g,kd+c] out[g,kd+c])  (softmax)
 *   gru_gate_bwd_indexed   gru_gate_bwd for gx [G,3H] picked up through node_to_graph_map: grad_gh [V,3H], grad_h_direct
 *                          [V,H] and grad_gx summed per graph to [G,3H] */
typedef enum {
  TFGNN_READOUT_SOFTMAX = 0,
  TFGNN_READOUT_SIGMOID = 1,
  TFGNN_READOUT_NONE = 2,
  TFGNN_READOUT_AVERAGE = 3
} tfgnn_readout_mode_t;
TFGNN_API int tfgnn_b200_segment_sum_rows(const float* data, const int32_t* node_to_graph_map, const int32_t* graph_ptr,
                                          int64_t num_rows, int32_t num_graphs, int32_t C, float* out, void* stream);
TFGNN_API int tfgnn_b200_readout_bwd(const float* node_reprs, const float* weights, const int32_t* node_to_graph_map,
                                     const int32_t* graph_ptr, const float* out, const float* grad_out, int64_t num_nodes,
                                     int32_t num_graphs, int32_t repr_dim, int32_t num_heads, int32_t mode, float lower,
                                     float upper, int32_t has_lower, int32_t has_upper, float* grad_reprs,
                                     float* grad_scores, void* stream);
TFGNN_API int tfgnn_b200_gru_gate_bwd_indexed(const float* gx, const int32_t* node_to_graph_map, const int32_t* graph_ptr,
                                              const float* gh, const float* h, const float* grad_out, int64_t num_rows,
                                              int32_t num_graphs, int32_t H, float* grad_gx, float* grad_gh,
                                              float* grad_h_direct, void* stream);

/* ---- On-device batch builder (SURVEY.md section 8f-2) ------------------------------------------------------
 * Bit-exact int32 bookkeeping of the data layer, so that a training loop never leaves the device between the
 * packed dataset and the layer call.
 *
 * process_adjacency_lists (tf2_gnn/data/utils.py:9-58): from the T forward edge lists [E_t,2] build the processed
 * lists: forward types first (a tied type gets its flipped edges appended, utils.py:102-108), then one fresh type
 * of flipped edges per untied forward type (:109-113), then, if add_self_loop_edges, the list (i,i) for all nodes
 * inserted at slot self_loop_edge_type (negative values count from the end, list.insert semantics of :91-99;
 * values outside [-(n+1), n] are TFGNN_ERR_INVALID_ARGUMENT like the reference's assert).
 *   tied                 host int32[T], non-zero = tie_fwd_bkwd for that forward type (get_tied_edge_types, :61-77)
 *   _sizes               host-only: number of processed types and their edge counts (compute_number_of_edge_types, :80-84)
 *   adjacency_out        host array of num_types_out caller-allocated device lists, sizes as reported by _sizes
 *   type_to_num_incoming_edges  optional float32[num_types_out, V]: in-degree per processed type (:116-124; the
 *                        reference returns float64 of the same integer values) */
TFGNN_API int tfgnn_b200_process_adjacency_sizes(const int64_t* num_edges_fwd, int32_t num_fwd_types, int64_t num_nodes,
                                       int32_t add_self_loop_edges, const int32_t* tied,
                                       int32_t self_loop_edge_type, int64_t* num_edges_out,
                                       int32_t* num_types_out);
TFGNN_API int tfgnn_b200_process_adjacency(const int32_t* const* adjacency_fwd, const int64_t* num_edges_fwd,
                                 int32_t num_fwd_types, int64_t num_nodes, int32_t add_self_loop_edges,
                                 const int32_t* tied, int32_t self_loop_edge_type,
                                 int32_t* const* adjacency_out, int32_t num_types_out,
                                 float* type_to_num_incoming_edges, void* stream);

/* Disjoint-union minibatch (GraphDataset._add_graph_to_batch / _finalise_batch, graph_dataset.py:161-246) from a
 * dataset stored packed on the device: node_offsets int64[G+1] (graph g owns rows [off[g], off[g+1]) of the node
 * table), and per edge type t edge_offsets[t] int64[G+1] into edges[t] int32[*,2] holding graph-local node ids.
 *   graph_ids            device int32[num_graphs_in_batch], in batch order
 *   num_nodes_in_batch, num_edges_in_batch[t]   sizes of the outputs (the host knows them from its copy of the
 *                        offset tables; larger values than the real totals are clamped on the device)
 *   node_to_graph_map    out int32[num_nodes_in_batch]: batch-local graph index of every node (:211-217), or NULL
 *   node_source_rows     out int32[num_nodes_in_batch]: row of every batch node in the packed node table (feed it to
 *                        tfgnn_b200_gather_rows to assemble node_features), or NULL
 *   adjacency_lists      host array of T caller-allocated device lists [num_edges_in_batch[t], 2]: stored pairs plus
 *                        the running node count of their graph (:218-222)
 *   workspace            device, tfgnn_b200_assemble_batch_workspace_bytes(T, num_graphs_in_batch) bytes */
TFGNN_API size_t tfgnn_b200_assemble_batch_workspace_bytes(int32_t num_edge_types, int32_t num_graphs_in_batch);
TFGNN_API int tfgnn_b200_assemble_batch(const int64_t* node_offsets, const int64_t* const* edge_offsets,
                              const int32_t* const* edges, int32_t num_edge_types, int64_t num_graphs_total,
                              const int32_t* graph_ids, int32_t num_graphs_in_batch,
                              int64_t num_nodes_in_batch, const int64_t* num_edges_in_batch,
                              int32_t* node_to_graph_map, int32_t* node_source_rows,
                              int32_t* const* adjacency_lists, void* workspace, void* stream);

/* ---- Device-global state --------------------------------------------------------------------------------------
 * Two things in this library outlive a call and are shared with the host framework's CUDA context:
 *   (1) the fused RGCN kernel keeps its hand-off ring and the packed weights resident in L2 with evict_last hints,
 *       which only bind inside a persisting-L2 carve-out.  The first fused launch on a device therefore saves the
 *       current cudaLimitPersistingL2CacheSize and raises it (never lowers it).  Default size: what the launch
 *       keeps resident (ring + packed weights + 4 MB), at least 72 MB, at most the device maximum, raised again by
 *       a later launch that needs more; set_l2_persist_mb(megabytes) fixes the size instead, set_l2_persist_mb(0)
 *       opts out (results identical, ~4 GB more HBM traffic per cfg2 layer); -1 returns to the default /
 *       TFGNN_B200_L2_PERSIST_MB.
 *   (2) a private stream-ordered memory pool (cudaMemPool) that caches the library's own buffers.
 * tfgnn_b200_release_device_state() restores the saved L2 limit on every device and trims the pool; the Python
 * shim registers it with atexit.
 * Threading: entry points are re-entrant; ONE tfgnn_batch_t must not be used by two host threads or on two
 * streams at the same time (it may move to another stream between calls: the library orders the streams). */
TFGNN_API int tfgnn_b200_set_l2_persist_mb(int32_t megabytes);
TFGNN_API int tfgnn_b200_release_device_state(void);

/* Number of kernels this library has launched in the calling process (all threads). */
TFGNN_API int64_t tfgnn_b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* TFGNN_B200_H_ */
