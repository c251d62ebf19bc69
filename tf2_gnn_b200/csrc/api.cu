// C-ABI entry points (include/tfgnn_b200.h): argument validation and the per-layer orchestration
// of the edge-level (HBM-bound) and node-level (tensor-core / FFMA) kernels.
//
// Formulations (exact in real arithmetic; fp32 reassociation only — DESIGN.md §3):
//   aggregate-then-transform  out = act( rn(v) * [A_0|..|A_{L-1}] [W_0;..;W_{L-1}] ),
//                             A_l[v] = 1/(c_{v,l}+eps) * sum_{(u,v) in A_l} h_u
//     valid when the message is linear in h_u and the aggregation is sum/mean/sqrt_n with the
//     activation after it (RGCN/GGNN defaults, every PPI/QM9 RGCN config).
//   transform-then-aggregate  P = h [W_0|..|W_{L-1}];  out[v] = agg_{l,e} f(P_l[src_e], v, l)
//     for max-aggregation / activation-before-aggregation (per-edge non-linearity); its backward
//     (backward.cu) recomputes P through the same transform_aggregate_tables and differentiates f per edge.
//   hoisted hidden layer      A_l[v] = scale * sum_e relu(U^s_l h_u + U^t_l h_v); out = act(A W2cat)
#include <cstdlib>
#include <mutex>
#include <string>

#include "layers.cuh"

namespace tfgnn {

std::atomic<long long> g_launch_count{0};
static thread_local std::string t_last_error;
static thread_local int t_last_code = 0;

void set_error(int code, const std::string& msg) {
  t_last_code = code;
  t_last_error = msg;
}
int last_error_code() { return t_last_code; }

int check_cuda(cudaError_t e, const char* what, const char* file, int line) {
  if (e == cudaSuccess) return 0;
  set_error(TFGNN_ERR_CUDA, std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what + " (" + file +
                                ":" + std::to_string(line) + ")");
  return TFGNN_ERR_CUDA;
}

int unsupported(const std::string& msg) {
  set_error(TFGNN_ERR_UNSUPPORTED, msg);
  return TFGNN_ERR_UNSUPPORTED;
}

bool valid_act(int a) { return a >= TFGNN_ACT_NONE && a <= TFGNN_ACT_SIGMOID; }
bool valid_agg(int a) { return a >= TFGNN_AGG_SUM && a <= TFGNN_AGG_SQRT_N; }

// Node-level contraction C = epi(A B) with B [K,N] row-major in device memory.  The tensor-core path packs B into a pool
// buffer freed after the GEMM.
int node_gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, long long M, int N, int K,
              const GemmEpilogue& epi, int path, cudaStream_t st) {
  const bool want_tc = (path == TFGNN_PATH_AUTO || path == TFGNN_PATH_SORTED_TC || path == TFGNN_PATH_FUSED_TC);
  const bool mul_ok = epi.mul == nullptr || (epi.ldm % 4 == 0 && (reinterpret_cast<uintptr_t>(epi.mul) & 15) == 0);
  const bool bias_ok = epi.bias == nullptr || (reinterpret_cast<uintptr_t>(epi.bias) & 15) == 0;   // float4 bias loads
  if (want_tc && mul_ok && bias_ok && gemm_tc_supported(M, N, K, A, lda, C, ldc)) {   // the packing kernel takes any ldb
    PoolBuffer packed{st};
    int rc = packed.alloc(gemm_tc_packed_bytes(N, K));
    if (!rc) rc = launch_pack_weights_tc(B, ldb, K, N, packed.f(), st);
    if (!rc) rc = launch_gemm_tc(A, lda, packed.f(), C, ldc, M, N, K, epi, st);
    return rc;
  }
  if (path == TFGNN_PATH_SORTED_TC)
    return unsupported("TFGNN_PATH_SORTED_TC: shape not supported by the tensor-core GEMM (need N%16==0, K%32==0)");
  return launch_gemm_simt(A, lda, B, ldb, C, ldc, M, N, K, epi, st);
}

static int pipeline_init(tfgnn_batch* b) {
  if (b->pipe_ready) return 0;
  int lo = 0, hi = 0;
  TFGNN_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  TFGNN_CUDA(cudaStreamCreateWithPriority(&b->pipe_gather, cudaStreamNonBlocking, lo));
  TFGNN_CUDA(cudaStreamCreateWithPriority(&b->pipe_gemm, cudaStreamNonBlocking, hi));
  TFGNN_CUDA(cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming));
  TFGNN_CUDA(cudaEventCreateWithFlags(&b->ev_join_g, cudaEventDisableTiming));
  TFGNN_CUDA(cudaEventCreateWithFlags(&b->ev_join_m, cudaEventDisableTiming));
  for (int i = 0; i < tfgnn_batch::kPipeBufs; ++i) {
    TFGNN_CUDA(cudaEventCreateWithFlags(&b->ev_g[i], cudaEventDisableTiming));
    TFGNN_CUDA(cudaEventCreateWithFlags(&b->ev_m[i], cudaEventDisableTiming));
  }
  b->pipe_ready = true;
  return 0;
}

// RGCN-style layer as a two-stream pipeline over node chunks: the HBM-bound gather/reduce of chunk
// i+1 (stream G) overlaps the tensor-core contraction of chunk i (stream M); the per-chunk
// intermediate A[chunk, L*D] is triple-buffered.  Fork/join on the caller's stream with events, so
// the call stays stream-ordered (and graph-capturable).
static int pipe_chunk_rows() {
  // default: two 128-row tiles per SM; TFGNN_B200_PIPE_CHUNK_ROWS overrides (tests / tuning)
  int rows = 2 * 132 * 128;
  if (const char* e = getenv("TFGNN_B200_PIPE_CHUNK_ROWS")) {
    const int v = atoi(e);
    if (v >= 128) rows = (v > (1 << 24) ? (1 << 24) : v) / 128 * 128;
  }
  return rows;
}
static int rgcn_pipelined(tfgnn_batch* b, const float* h, int D, const float* Wcat, int H, bool normalize,
                          const GemmEpilogue& epi_in, float* out, int ldo, cudaStream_t st) {
  const int V = (int)b->V, L = b->L, K = L * D;
  const int kPipeChunkRows = pipe_chunk_rows();
  int rc = pipeline_init(b);
  if (rc) return rc;
  // A and the packed weights are allocated on `st` before the fork and freed on `st` by their destructors when this
  // function returns, after `st` has waited on both join events: the frees are ordered after the last chunk on G and M.
  // A failed launch inside the loop therefore still leaves through the join.
  const size_t a_chunk_elems = (size_t)kPipeChunkRows * K;
  PoolBuffer A{st}, packed{st};
  rc = A.alloc(a_chunk_elems * tfgnn_batch::kPipeBufs * sizeof(float));
  if (!rc) rc = packed.alloc(gemm_tc_packed_bytes(H, K));
  if (!rc) rc = launch_pack_weights_tc(Wcat, H, K, H, packed.f(), st);
  if (rc) return rc;
  cudaStream_t sg = b->pipe_gather, sm = b->pipe_gemm;
  TFGNN_CUDA(cudaEventRecord(b->ev_fork, st));
  TFGNN_CUDA(cudaStreamWaitEvent(sg, b->ev_fork, 0));
  TFGNN_CUDA(cudaStreamWaitEvent(sm, b->ev_fork, 0));
  const int nchunks = (V + kPipeChunkRows - 1) / kPipeChunkRows;
  for (int i = 0; i < nchunks; ++i) {
    const int buf = i % tfgnn_batch::kPipeBufs;
    const int v0 = i * kPipeChunkRows;
    const int vc = (V - v0 < kPipeChunkRows) ? V - v0 : kPipeChunkRows;
    float* Abuf = A.f() + (size_t)buf * a_chunk_elems;
    if (i >= tfgnn_batch::kPipeBufs) TFGNN_CUDA(cudaStreamWaitEvent(sg, b->ev_m[buf], 0));
    EdgeReduceParams p;
    p.X = h; p.ldx = D; p.x_type_stride = 0;
    p.row_ptr = b->row_ptr; p.src = b->src_sorted;
    p.out = Abuf; p.ldo = K; p.out_type_stride = D;
    p.V = V; p.L = L; p.C = D; p.normalize = normalize;
    p.v_begin = v0; p.v_count = vc;
    static const int gather_cap = [] {
      const char* e = getenv("TFGNN_B200_PIPE_GATHER_BLOCKS");
      return e && atoi(e) > 0 ? atoi(e) : 132 * 3;   // 3 lean CTAs/SM leave registers for the GEMM CTA
    }();
    rc = launch_edge_reduce(p, /*merged=*/false, sg, gather_cap);
    if (rc) break;
    TFGNN_CUDA(cudaEventRecord(b->ev_g[buf], sg));
    TFGNN_CUDA(cudaStreamWaitEvent(sm, b->ev_g[buf], 0));
    GemmEpilogue epi = epi_in;
    epi.row0 = v0;
    rc = launch_gemm_tc(Abuf, K, packed.f(), out + (size_t)v0 * ldo, ldo, vc, H, K, epi, sm);
    if (rc) break;
    TFGNN_CUDA(cudaEventRecord(b->ev_m[buf], sm));
  }
  TFGNN_CUDA(cudaEventRecord(b->ev_join_g, sg));
  TFGNN_CUDA(cudaEventRecord(b->ev_join_m, sm));
  TFGNN_CUDA(cudaStreamWaitEvent(st, b->ev_join_g, 0));
  TFGNN_CUDA(cudaStreamWaitEvent(st, b->ev_join_m, 0));
  return rc;
}

int agg_row_norm(int aggregation) {
  return aggregation == TFGNN_AGG_MEAN ? 1 : aggregation == TFGNN_AGG_SQRT_N ? 2 : 0;
}

// The node-level half of the transform-then-aggregate form (no hidden layer; max aggregation and / or activation before
// aggregation): P = h [W_0|..|W_{L-1}] over the Vs source rows and, with target-state input, T = h_tgt [W^t_0|..] over the
// owned rows, W_l = W.p[l], into the caller's buffers.  *p becomes the merged edge reduce that forms the layer from them,
// out / ldo unset:  out[v] = act_final(agg_e act_edge((P_l[u] + T_l[v]) s)).  The backward recomputes both through this
// function.
int transform_aggregate_tables(tfgnn_batch* b, const float* h, int D, const PtrTable& W, int H, uint32_t flags,
                               int aggregation, int activation, int path, PoolBuffer& P, PoolBuffer& T,
                               EdgeReduceParams* p, cudaStream_t st) {
  const int V = (int)b->V, Vs = (int)b->V_src, L = b->L, LH = L * H;
  const bool act_before = flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION;
  PoolBuffer Wcat{st};
  int rc = P.alloc((size_t)Vs * LH * sizeof(float));
  if (!rc) rc = Wcat.alloc((size_t)D * LH * sizeof(float));
  if (!rc) rc = launch_pack_horizontal(W, L, 0, D, H, H, Wcat.f(), LH, st);
  if (rc) return rc;
  GemmEpilogue none;
  rc = node_gemm(h, D, Wcat.f(), LH, P.f(), LH, Vs, LH, D, none, path, st);
  if (rc) return rc;
  if (flags & TFGNN_FLAG_USE_TARGET_STATE) {
    rc = T.alloc((size_t)V * LH * sizeof(float));
    if (!rc) rc = launch_pack_horizontal(W, L, D, D, H, H, Wcat.f(), LH, st);
    if (!rc) rc = node_gemm(h + (size_t)b->tgt_off * D, D, Wcat.f(), LH, T.f(), LH, V, LH, D, none, path, st);
    if (rc) return rc;
  }
  *p = EdgeReduceParams{};
  p->X = P.f(); p->ldx = LH; p->x_type_stride = H;
  p->T = T.f(); p->ldt = LH; p->t_type_stride = H;
  p->row_ptr = b->row_ptr; p->src = b->src_sorted;
  p->V = V; p->L = L; p->C = H;
  p->normalize = (flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING) != 0;
  p->edge_act = act_before ? activation : TFGNN_ACT_NONE;
  p->reduce_max = aggregation == TFGNN_AGG_MAX;
  p->row_norm = agg_row_norm(aggregation);
  p->final_act = act_before ? TFGNN_ACT_NONE : activation;
  return 0;
}

// Edge-MLP family core.  Writes act/agg result to out[V, ldo].
int edge_mlp_core(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights,
                         int n_hidden, int H, uint32_t flags, int aggregation, int activation, int path,
                         float* out, int ldo, cudaStream_t st) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  TFGNN_REQUIRE(D > 0 && H > 0, "D and H must be positive");
  TFGNN_REQUIRE(n_hidden >= 0, "num_hidden_layers must be >= 0");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  TFGNN_REQUIRE(valid_agg(aggregation), "unknown aggregation code");
  TFGNN_REQUIRE(path >= TFGNN_PATH_AUTO && path <= TFGNN_PATH_FUSED_TC, "unknown path code");
  const int V = (int)b->V, L = b->L;
  const int Vs = (int)b->V_src;                           // rows of the source table h
  if (V == 0) return 0;
  {
    const int rc_enter = batch_enter(b, st);
    if (rc_enter) return rc_enter;
  }
  TFGNN_REQUIRE(h != nullptr && out != nullptr, "h / out is NULL");
  TFGNN_REQUIRE(L == 0 || mlp_weights != nullptr, "mlp_weights is NULL");
  const float* h_tgt = h + (size_t)b->tgt_off * D;        // rows of the targets owned by this batch
  const bool sharded = (b->tgt_off != 0 || b->V_src != b->V);
  const int n_layers = n_hidden + 1;
  for (int i = 0; i < L * n_layers; ++i) TFGNN_REQUIRE(mlp_weights[i] != nullptr, "a weight pointer is NULL");

  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const bool act_before = flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;
  const bool sum_like = aggregation != TFGNN_AGG_MAX;
  const int row_norm = agg_row_norm(aggregation);

  PtrTable first{}, last{};
  for (int l = 0; l < L; ++l) {
    first.p[l] = mlp_weights[l * n_layers];
    last.p[l] = mlp_weights[l * n_layers + n_hidden];
  }

  if (b->n_peer_out > 0 && !(L > 0 && n_hidden == 0 && sum_like && !act_before && !use_target))
    return unsupported("rgcn_fwd_allgather needs an RGCN-style layer (linear messages, sum/mean/sqrt_n, activation after)");
  if (L == 0) {
    // No edges at all: agg identity then activation (message_passing.py:172-177).
    EdgeReduceParams p;
    p.X = h; p.ldx = D; p.row_ptr = b->row_ptr; p.src = b->src_sorted;
    p.out = out; p.ldo = ldo; p.V = V; p.L = 0; p.C = H;
    p.reduce_max = aggregation == TFGNN_AGG_MAX;
    p.final_act = act_before ? TFGNN_ACT_NONE : activation;
    return launch_edge_reduce(p, /*merged=*/true, st);
  }

  if (n_hidden == 0 && sum_like && !act_before) {
    // ---- aggregate-then-transform ----
    const int K = L * D * (use_target ? 2 : 1);
    const bool pipelined = (path == TFGNN_PATH_AUTO || path == TFGNN_PATH_FUSED_TC) && !use_target &&
                           V >= 2 * pipe_chunk_rows() && D % 4 == 0 &&
                           gemm_tc_supported(V, H, K, h, K, out, ldo) &&
                           (reinterpret_cast<uintptr_t>(h) & 15) == 0;
    const bool fused_ok = !use_target && fused_rgcn_supported(V, L, D, H, h, out, ldo);
    if (path == TFGNN_PATH_FUSED_TC && !fused_ok)
      return unsupported("TFGNN_PATH_FUSED_TC needs D % 32 == 0, 16 <= H <= 512 (H % 16 == 0; H > 64: <= 7 edge types), no target-state input");
    static const bool fused_auto = [] { const char* e = getenv("TFGNN_B200_FUSED"); return !e || atoi(e) != 0; }();
    if (fused_ok && (path == TFGNN_PATH_FUSED_TC || (path == TFGNN_PATH_AUTO && fused_auto))) {
      PoolBuffer packed{st}, ring{st};
      const int corr = fused_corr_bf16(activation);
      int rc = packed.alloc(gemm_tc_packed_bytes(H, K));
      if (!rc) rc = ring.alloc(fused_rgcn_ring_bytes(D, L, H));
      if (!rc) rc = launch_pack_weights_tc_table(first, L, D, H, corr, packed.f(), st);   // [W_0;..;W_{L-1}] -> K-major hi / correction
      if (rc) return rc;
      GemmEpilogue epi;
      epi.act = activation;
      epi.row_norm = row_norm; epi.row_ptr = b->row_ptr; epi.V = V; epi.L = L;
      if (b->ln_gamma && fused_rgcn_ln_supported(H)) {   // LayerNorm in the epilogue; the caller is told through ln_done
        epi.ln_gamma = b->ln_gamma; epi.ln_beta = b->ln_beta; epi.ln_eps = b->ln_eps;
        b->ln_gamma = nullptr;         // consumed
      }
      return launch_fused_rgcn(h, D, b->row_ptr, b->src_sorted, b->M_in, V, L, normalize, packed.f(), corr, H, ring.f(),
                               out, ldo, epi, st, b->peer_out, b->n_peer_out, b->mc_out);
    }
    if (b->n_peer_out > 0)
      return unsupported("rgcn_fwd_allgather: this shard does not take the fused kernel (need D % 32 == 0, 16 <= H <= 512, "
                         "H % 16 == 0, no target-state input)");
    PoolBuffer Wcat{st};
    int rc = Wcat.alloc((size_t)K * H * sizeof(float));
    if (rc) return rc;
    if (pipelined) {
      rc = launch_pack_vertical(first, L, 0, D, H, H, Wcat.f(), H, 0, st);
      if (rc) return rc;
      GemmEpilogue epi;
      epi.act = activation;
      epi.row_norm = row_norm; epi.row_ptr = b->row_ptr; epi.V = V; epi.L = L;
      return rgcn_pipelined(b, h, D, Wcat.f(), H, normalize, epi, out, ldo, st);
    }
    PoolBuffer A{st};
    rc = A.alloc((size_t)V * K * sizeof(float));
    if (rc) return rc;
    if (path == TFGNN_PATH_ATOMIC) {
      if (sharded) return unsupported("TFGNN_PATH_ATOMIC is not available on a target-range shard");
      TFGNN_CUDA(cudaMemsetAsync(A.p, 0, (size_t)V * K * sizeof(float), st));
      rc = launch_edge_scatter_atomic(b, h, D, D, normalize, A.f(), K, D, st);
      if (rc) return rc;
    } else {
      EdgeReduceParams p;
      p.X = h; p.ldx = D; p.x_type_stride = 0;
      p.row_ptr = b->row_ptr; p.src = b->src_sorted;
      p.out = A.f(); p.ldo = K; p.out_type_stride = D;
      p.V = V; p.L = L; p.C = D; p.normalize = normalize;
      rc = launch_edge_reduce(p, /*merged=*/false, st);
      if (rc) return rc;
    }
    rc = launch_pack_vertical(first, L, 0, D, H, H, Wcat.f(), H, 0, st);
    if (rc) return rc;
    if (use_target) {
      rc = launch_target_term(h_tgt, D, b->row_ptr, V, L, D, normalize, A.f(), K, L * D, st);
      if (rc) return rc;
      rc = launch_pack_vertical(first, L, D, D, H, H, Wcat.f(), H, L * D, st);
      if (rc) return rc;
    }
    GemmEpilogue epi;
    epi.act = activation;
    epi.row_norm = row_norm; epi.row_ptr = b->row_ptr; epi.V = V; epi.L = L;
    return node_gemm(A.f(), K, Wcat.f(), H, out, ldo, V, H, K, epi, path, st);
  }

  if (path == TFGNN_PATH_ATOMIC)
    return unsupported("TFGNN_PATH_ATOMIC only implements the linear-message sum/mean/sqrt_n case");

  if (n_hidden == 0) {
    // ---- transform-then-aggregate (max aggregation and/or activation before aggregation) ----
    EdgeReduceParams p;
    PoolBuffer P{st}, T{st};
    int rc = transform_aggregate_tables(b, h, D, first, H, flags, aggregation, activation, path, P, T, &p, st);
    if (rc) return rc;
    p.out = out; p.ldo = ldo;
    return launch_edge_reduce(p, /*merged=*/true, st);
  }

  if (n_hidden == 1 && sum_like && !act_before) {
    // ---- hoisted hidden layer: per-edge relu on pre-projected tables, output layer per (v,l) ----
    const int LH = L * H;
    PoolBuffer Xs{st}, Xt{st}, A{st}, W2{st};
    int rc = Xs.alloc((size_t)Vs * LH * sizeof(float));
    if (rc) return rc;
    {
      PoolBuffer Wcat{st};
      rc = Wcat.alloc((size_t)D * LH * sizeof(float));
      if (!rc) rc = launch_pack_horizontal(first, L, 0, D, H, H, Wcat.f(), LH, st);
      if (rc) return rc;
      GemmEpilogue none;
      rc = node_gemm(h, D, Wcat.f(), LH, Xs.f(), LH, Vs, LH, D, none, path, st);
      if (rc) return rc;
      if (use_target) {
        rc = Xt.alloc((size_t)V * LH * sizeof(float));
        if (!rc) rc = launch_pack_horizontal(first, L, D, D, H, H, Wcat.f(), LH, st);
        if (!rc) rc = node_gemm(h_tgt, D, Wcat.f(), LH, Xt.f(), LH, V, LH, D, none, path, st);
        if (rc) return rc;
      }
    }
    rc = A.alloc((size_t)V * LH * sizeof(float));
    if (rc) return rc;
    EdgeReduceParams p;
    p.X = Xs.f(); p.ldx = LH; p.x_type_stride = H;
    p.T = Xt.f(); p.ldt = LH; p.t_type_stride = H;
    p.row_ptr = b->row_ptr; p.src = b->src_sorted;
    p.out = A.f(); p.ldo = LH; p.out_type_stride = H;
    p.V = V; p.L = L; p.C = H; p.normalize = normalize; p.hidden_relu = 1;
    rc = launch_edge_reduce(p, /*merged=*/false, st);
    if (!rc) rc = W2.alloc((size_t)LH * H * sizeof(float));
    if (!rc) rc = launch_pack_vertical(last, L, 0, H, H, H, W2.f(), H, 0, st);
    if (rc) return rc;
    GemmEpilogue epi;
    epi.act = activation;
    epi.row_norm = row_norm; epi.row_ptr = b->row_ptr; epi.V = V; epi.L = L;
    return node_gemm(A.f(), LH, W2.f(), H, out, ldo, V, H, LH, epi, path, st);
  }

  // edge MLP with >= 2 hidden layers, or hidden layers combined with max-aggregation /
  // activation-before-aggregation: the per-edge non-linearity cannot be hoisted -> literal path.
  return edge_mlp_literal(b, h, D, mlp_weights, n_hidden, H, flags, aggregation, activation, nullptr, 0, path, out,
                          ldo, st);
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_abi_version(void) { return TFGNN_B200_ABI_VERSION; }
extern "C" const char* tfgnn_b200_last_error(void) { return t_last_error.c_str(); }
extern "C" int64_t tfgnn_b200_launch_count(void) { return g_launch_count.load(); }
extern "C" int tfgnn_b200_set_l2_persist_mb(int32_t megabytes) { return set_l2_persist_mb(megabytes); }
extern "C" int tfgnn_b200_release_device_state(void) {
  restore_l2_persist_carveout();
  pool_trim_all();
  return 0;
}

extern "C" int tfgnn_b200_edge_mlp_fwd(tfgnn_batch_t* batch, const float* h, int32_t D,
                                       const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H,
                                       uint32_t flags, int32_t aggregation, int32_t activation, int32_t path,
                                       float* out, void* stream) {
  return edge_mlp_core(batch, h, D, mlp_weights, num_hidden_layers, H, flags, aggregation, activation, path, out,
                       H, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_rgcn_fwd(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W,
                                   int32_t H, uint32_t flags, int32_t aggregation, int32_t activation,
                                   int32_t path, float* out, void* stream) {
  return edge_mlp_core(batch, h, D, W, 0, H, flags & ~TFGNN_FLAG_USE_TARGET_STATE, aggregation, activation, path,
                       out, H, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_rgcn_fwd_allgather(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W,
                                             int32_t H, uint32_t flags, int32_t aggregation, int32_t activation,
                                             float* const* out_replicas, int32_t num_replicas, int32_t own_rank,
                                             float* out_multicast, void* stream) {
  TFGNN_REQUIRE(batch != nullptr, "batch is NULL");
  TFGNN_REQUIRE(out_replicas != nullptr && num_replicas >= 1 && num_replicas <= TFGNN_MAX_PEERS + 1,
                "num_replicas must be in [1, 16]");
  TFGNN_REQUIRE(own_rank >= 0 && own_rank < num_replicas, "own_rank out of range");
  for (int r = 0; r < num_replicas; ++r) TFGNN_REQUIRE(out_replicas[r] != nullptr, "a replica pointer is NULL");
  // replica tables hold ALL nodes; the kernel indexes rows of the shard: shift every base to the shard's first row
  const size_t off = (size_t)batch->tgt_off * (size_t)H;
  int n = 0;
  for (int r = 0; r < num_replicas; ++r)
    if (r != own_rank) batch->peer_out[n++] = out_replicas[r] + off;
  batch->n_peer_out = n;   // 0 for a single replica: the plain fused layer
  batch->mc_out = (out_multicast && n > 0) ? out_multicast + off : nullptr;
  const int rc = edge_mlp_core(batch, h, D, W, 0, H, flags & ~TFGNN_FLAG_USE_TARGET_STATE, aggregation, activation,
                               TFGNN_PATH_FUSED_TC, out_replicas[own_rank] + off, H, (cudaStream_t)stream);
  batch->n_peer_out = 0;
  batch->mc_out = nullptr;
  return rc;
}

extern "C" int tfgnn_b200_layer_norm(const float* x, const float* gamma, const float* beta, int64_t V, int32_t H,
                                     float epsilon, float* out, void* stream);

extern "C" int tfgnn_b200_rgcn_ln_fwd(tfgnn_batch_t* batch, const float* h, int32_t D, const float* const* W, int32_t H,
                                      uint32_t flags, int32_t aggregation, int32_t activation, int32_t path,
                                      const float* ln_gamma, const float* ln_beta, float ln_epsilon, float* out,
                                      void* stream) {
  TFGNN_REQUIRE(batch != nullptr, "batch is NULL");
  TFGNN_REQUIRE(ln_gamma && ln_beta, "LayerNorm parameter pointer is NULL");
  const bool aligned = ((reinterpret_cast<uintptr_t>(ln_gamma) | reinterpret_cast<uintptr_t>(ln_beta)) & 15) == 0;
  if (aligned) {
    batch->ln_gamma = ln_gamma; batch->ln_beta = ln_beta; batch->ln_eps = ln_epsilon;
  }
  int rc = edge_mlp_core(batch, h, D, W, 0, H, flags & ~TFGNN_FLAG_USE_TARGET_STATE, aggregation, activation, path, out, H,
                         (cudaStream_t)stream);
  const bool fused = aligned && batch->ln_gamma == nullptr;   // the fused kernel consumed the parameters
  batch->ln_gamma = nullptr; batch->ln_beta = nullptr;
  if (rc || fused) return rc;
  // shapes the fused kernel does not take (H > 64, split-tile batches are handled inside, unaligned parameters, other
  // paths): same result from the stand-alone kernel, in place
  return tfgnn_b200_layer_norm(out, ln_gamma, ln_beta, batch->V, H, ln_epsilon, out, stream);
}

extern "C" int tfgnn_b200_dense_fwd(const float* x, const float* W, float* out, int64_t V, int32_t K, int32_t N,
                                    int32_t activation, int32_t path, void* stream) {
  TFGNN_REQUIRE(V >= 0 && K > 0 && N > 0, "bad dense shape");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  if (V == 0) return 0;
  TFGNN_REQUIRE(x && W && out, "NULL pointer");
  GemmEpilogue epi;
  epi.act = activation;
  return node_gemm(x, K, W, N, out, N, V, N, K, epi, path, (cudaStream_t)stream);
}
