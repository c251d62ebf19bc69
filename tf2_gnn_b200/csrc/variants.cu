// GGNN / RGIN / GNN-FiLM / RGAT entry points: compositions of the edge-level and node-level kernels.
#include "layers.cuh"

namespace tfgnn {

// Keras GRUCell, reset_after=True (ggnn.py:84-87): gx = agg K + b0, gh = h U + b1 (both [V,3H]),
// z = sigmoid(gx_z+gh_z), r = sigmoid(gx_r+gh_r), hh = tanh(gx_h + r*gh_h), h' = z*h + (1-z)*hh.
// gx_index (optional) picks row gx_index[v] of gx for row v: the GRU exchange computes graph_repr K + b0 once per GRAPH.
// out may overlap h (an in-place state update): each thread reads its h element before it writes.
__global__ void gru_gate_kernel(const float* __restrict__ gx, const int* __restrict__ gx_index,
                                const float* __restrict__ gh, const float* h, int ldh, long long V, int H, float* out) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    const int c = (int)(i - v * H);
    const float* x = gx + (gx_index ? (long long)__ldg(gx_index + v) : v) * 3 * H;
    const float* r_ = gh + v * 3 * H;
    const float z = 1.0f / (1.0f + expf(-(x[c] + r_[c])));
    const float r = 1.0f / (1.0f + expf(-(x[H + c] + r_[H + c])));
    const float hh = tanhf(x[2 * H + c] + r * r_[2 * H + c]);
    const float hp = h[v * ldh + c];
    out[i] = z * hp + (1.0f - z) * hh;
  }
}

int gru_update(const float* agg, const float* h, int ldh, const float* gru_kernel, const float* gru_recurrent_kernel,
               const float* gru_bias, long long V, int H, int path, bool in_place, float* out, cudaStream_t st) {
  {
    // The GRU update as ONE tensor-core contraction over [agg | h] with the gate math in its epilogue: no [V,3H] tables.
    // TFGNN_B200_GGNN_FUSED_GRU=0 keeps the two GEMMs + gate kernel (read per call: the tests compare the two).
    const char* e = getenv("TFGNN_B200_GGNN_FUSED_GRU");
    const bool want = !(e && atoi(e) == 0) &&
                      (path == TFGNN_PATH_AUTO || path == TFGNN_PATH_SORTED_TC || path == TFGNN_PATH_FUSED_TC);
    // the contraction reads whole rows of h for every 32-unit column tile while earlier tiles' epilogues already store new
    // states: an in-place update (the gate kernel below tolerates it) must not take this form
    if (want && !in_place && gemm_tc_gru_supported(V, H, agg, H, h, ldh, out, H)) {
      PoolBuffer packed{st};
      int rc = packed.alloc(gemm_tc_gru_packed_bytes(H));
      if (rc) return rc;
      return launch_gemm_tc_gru(agg, H, h, ldh, gru_kernel, gru_recurrent_kernel, gru_bias, packed.f(), out, H, V, H, st);
    }
  }
  PoolBuffer gx{st}, gh{st};
  int rc = gx.alloc((size_t)V * 3 * H * sizeof(float));
  if (!rc) rc = gh.alloc((size_t)V * 3 * H * sizeof(float));
  if (rc) return rc;
  GemmEpilogue ex, eh;
  ex.bias = gru_bias;
  eh.bias = gru_bias + 3 * H;
  rc = node_gemm(agg, H, gru_kernel, 3 * H, gx.f(), 3 * H, V, 3 * H, H, ex, path, st);
  if (rc) return rc;
  rc = node_gemm(h, ldh, gru_recurrent_kernel, 3 * H, gh.f(), 3 * H, V, 3 * H, H, eh, path, st);
  if (rc) return rc;
  gru_gate_kernel<<<grid_for(V * H), 256, 0, st>>>(gx.f(), nullptr, gh.f(), h, ldh, V, H, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_gru_update_fwd(const float* agg, const float* h, int64_t num_rows, int32_t H,
                                         const float* gru_kernel, const float* gru_recurrent_kernel, const float* gru_bias,
                                         int32_t path, float* out, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && H > 0, "bad gru_update sizes");
  TFGNN_REQUIRE(path >= TFGNN_PATH_AUTO && path <= TFGNN_PATH_FUSED_TC, "unknown path code");
  if (path == TFGNN_PATH_ATOMIC) return unsupported("TFGNN_PATH_ATOMIC is not available for the GRU update");
  if (num_rows == 0) return 0;
  TFGNN_REQUIRE(agg && h && out, "NULL pointer");
  TFGNN_REQUIRE(gru_kernel && gru_recurrent_kernel && gru_bias, "GRU weight pointer is NULL");
  const bool in_place = out < h + (size_t)num_rows * H && h < out + (size_t)num_rows * H;   // out overlaps the state rows
  return gru_update(agg, h, H, gru_kernel, gru_recurrent_kernel, gru_bias, num_rows, H, path, in_place, out,
                    (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_ggnn_fwd(tfgnn_batch_t* b, const float* h, int32_t D, const float* const* mlp_weights,
                                   int32_t num_hidden_layers, int32_t H, uint32_t flags, int32_t aggregation,
                                   const float* gru_kernel, const float* gru_recurrent_kernel,
                                   const float* gru_bias, int32_t path, float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  TFGNN_REQUIRE(D == H, "GGNN needs node embedding dimension == hidden_dim (ggnn.py:30)");
  const long long V = b->V;
  if (V == 0) return 0;
  TFGNN_REQUIRE(gru_kernel && gru_recurrent_kernel && gru_bias, "GRU weight pointer is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = batch_enter(b, st);
  if (rc) return rc;
  PoolBuffer agg{st};
  rc = agg.alloc((size_t)V * H * sizeof(float));
  if (rc) return rc;
  // ggnn.py:68-89: aggregation of the messages, no activation (act_before is ignored too).
  rc = edge_mlp_core(b, h, D, mlp_weights, num_hidden_layers, H, flags & ~TFGNN_FLAG_ACT_BEFORE_AGGREGATION,
                     aggregation, TFGNN_ACT_NONE, path, agg.f(), H, st);
  if (rc) return rc;
  const bool in_place = out < h + (size_t)b->V_src * D && h < out + (size_t)V * H;   // out overlaps the state table
  return gru_update(agg.f(), h + (size_t)b->tgt_off * D, D, gru_kernel, gru_recurrent_kernel, gru_bias, V, H, path, in_place,
                    out, st);
}

extern "C" int tfgnn_b200_gru_gate_fwd(const float* gx, const int32_t* gx_row_index, const float* gh, const float* h,
                                       int64_t num_rows, int32_t H, float* out, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && H > 0, "bad gru_gate sizes");
  if (num_rows == 0) return 0;
  TFGNN_REQUIRE(gx && gh && h && out, "NULL pointer");
  gru_gate_kernel<<<grid_for(num_rows * H), 256, 0, (cudaStream_t)stream>>>(gx, gx_row_index, gh, h, H, num_rows, H, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_rgin_fwd(tfgnn_batch_t* b, const float* h, int32_t D, const float* const* mlp_weights,
                                   int32_t num_hidden_layers, int32_t H, uint32_t flags, int32_t aggregation,
                                   int32_t activation, const float* const* aggr_weights, int32_t num_aggr_layers,
                                   int32_t path, float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  TFGNN_REQUIRE(num_aggr_layers >= 0, "num_aggr_layers must be >= 0");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  cudaStream_t st = (cudaStream_t)stream;
  const long long V = b->V;
  // rgin.py:88-106: aggregate, optional MLP, then the activation (activation-before is ignored).
  flags &= ~TFGNN_FLAG_ACT_BEFORE_AGGREGATION;
  if (num_aggr_layers == 0)
    return edge_mlp_core(b, h, D, mlp_weights, num_hidden_layers, H, flags, aggregation, activation, path, out, H,
                         st);
  TFGNN_REQUIRE(aggr_weights != nullptr, "aggr_weights is NULL");
  if (V == 0) return 0;
  int rc = batch_enter(b, st);
  if (rc) return rc;
  PoolBuffer t0{st}, t1{st};
  rc = t0.alloc((size_t)V * H * sizeof(float));
  if (!rc) rc = t1.alloc((size_t)V * H * sizeof(float));
  if (!rc) rc = edge_mlp_core(b, h, D, mlp_weights, num_hidden_layers, H, flags, aggregation, TFGNN_ACT_NONE, path, t0.f(),
                              H, st);
  if (rc) return rc;
  float* cur = t0.f();
  float* nxt = t1.f();
  for (int i = 0; i < num_aggr_layers; ++i) {
    TFGNN_REQUIRE(aggr_weights[i] != nullptr, "an aggregation MLP weight pointer is NULL");
    const bool last = i == num_aggr_layers - 1;
    GemmEpilogue epi;
    epi.act = last ? activation : TFGNN_ACT_RELU;
    float* dst = last ? out : nxt;
    rc = node_gemm(cur, H, aggr_weights[i], H, dst, H, V, H, H, epi, path, st);
    if (rc) return rc;
    float* t = cur; cur = nxt; nxt = t;
    if (!last) cur = dst;
  }
  return 0;
}

namespace tfgnn {

// GNN-FiLM forward (gnn_film.py:83-108) with its FiLM MLPs' last layer fed from `fin` (the owned targets' rows): type l
// reads columns [l*fstride, l*fstride + S) through film_weights[l] [S, 2H]; fin has L*S columns.  fstride 0: every type
// reads the same S = D columns of the layer's own target state (tfgnn_b200_film_fwd; fin then has D columns).  The scalar
// arguments and fin are checked by the entries.
int film_fwd_core(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights, int num_hidden_layers,
                  const float* fin, int fstride, int S, const float* const* film_weights, int H, uint32_t flags,
                  int aggregation, int activation, int path, float* out, cudaStream_t st) {
  const int V = (int)b->V, L = b->L;
  if (V == 0) return 0;
  if (L == 0) return edge_mlp_core(b, h, D, mlp_weights, 0, H, flags, aggregation, activation, path, out, H, st);
  TFGNN_REQUIRE(mlp_weights && film_weights, "weight table is NULL");
  TFGNN_REQUIRE(num_hidden_layers >= 0, "num_hidden_layers must be >= 0");
  TFGNN_REQUIRE((long long)L * S < (1ll << 31), "L * S overflows");
  const int ldf = fstride ? L * S : D;   // columns of fin
  if (path == TFGNN_PATH_ATOMIC) return unsupported("TFGNN_PATH_ATOMIC is not available for GNN-FiLM");
  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const bool act_before = flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;
  const int LH = L * H;
  PtrTable first{}, film{};
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(mlp_weights[l * (num_hidden_layers + 1)] && film_weights[l], "a weight pointer is NULL");
    first.p[l] = mlp_weights[l * (num_hidden_layers + 1)];
    film.p[l] = film_weights[l];
  }
  const int Vs = (int)b->V_src;
  const float* h_tgt = h + (size_t)b->tgt_off * D;
  GemmEpilogue none;
  int rc = batch_enter(b, st);
  if (rc) return rc;
  // TFGNN_B200_FILM_ATT: 1 = always, 0 = never, unset = on target-range shards (where the projected-table form would
  // project all num_nodes_total sources on every rank) and when the projected tables would not fit comfortably
  const char* film_att_str = getenv("TFGNN_B200_FILM_ATT");   // read per call: the tests sweep it
  const int film_att_env = film_att_str ? atoi(film_att_str) : -1;
  const bool sharded_batch = b->tgt_off != 0 || b->V_src != b->V;
  const size_t projected_bytes = ((size_t)b->V_src * L * H + (size_t)V * 2 * L * H) * sizeof(float);
  const bool film_att = film_att_env >= 0 ? film_att_env != 0 : (sharded_batch || projected_bytes > ((size_t)20 << 30));   // a quarter of 80 GB
  if (film_att && num_hidden_layers == 0 && aggregation != TFGNN_AGG_MAX && !act_before && D % 4 == 0 && H % 4 == 0 &&
      S % 4 == 0 && ldf % 4 == 0 && (reinterpret_cast<uintptr_t>(h) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(fin) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    // ---- aggregate-then-transform ---------------------------------------------------------------------------
    // Every per-edge quantity of gnn_film.py:83-108 but h_u depends on (target, type) only, so
    //   sum_{e in A_l -> v} gamma_l(v) * (s W_l h_u [+ s W^t_l h_v]) + beta_l(v)
    //     = gamma_l(v) * (A_l[v] W_l [+ coeff_l(v) h_v W^t_l]) + c_{v,l} beta_l(v),        A_l[v] = s sum_e h_u,
    // with s = 1/(c+eps) or 1, coeff = c s.  The per-edge work is the plain row gather (edge_reduce, HBM-bound, exactly
    // the RGCN traffic); everything else is node-level contractions chained through the GEMM epilogue
    // (C += gamma * acc): no [V, L*H] projected table, no [V, 2*L*H] FiLM table, and on a target-range shard only
    // the OWNED rows are ever multiplied (the transform-then-aggregate form projects all num_nodes_total sources on
    // every rank: 123 GB per rank at BASELINE config 5).
    const int K = L * D, KB = L * S;   // columns of A (and of the target-state operand), of the beta operand
    PoolBuffer A{st}, T{st};
    rc = A.alloc((size_t)V * K * sizeof(float));
    if (!rc) rc = T.alloc((size_t)V * (K > KB ? K : KB) * sizeof(float));
    if (rc) return rc;
    {
      EdgeReduceParams p;
      p.X = h; p.ldx = D; p.x_type_stride = 0;
      p.row_ptr = b->row_ptr; p.src = b->src_sorted;
      p.out = A.f(); p.ldo = K; p.out_type_stride = D;
      p.V = V; p.L = L; p.C = D; p.normalize = normalize;
      rc = launch_edge_reduce(p, /*merged=*/false, st);
      if (rc) return rc;
    }
    // beta part: out = [c_0 z_0 | .. | c_{L-1} z_{L-1}] [Fbeta_0; ..; Fbeta_{L-1}] with z_l = type l's FiLM input (h_v for
    // fstride 0): one L*S contraction, not finalised
    rc = launch_target_term(fin, ldf, b->row_ptr, V, L, S, /*normalize=*/0, T.f(), KB, 0, st, fstride);
    if (rc) return rc;
    {
      PoolBuffer Fb{st};
      PtrTable fbeta{};
      for (int l = 0; l < L; ++l) fbeta.p[l] = reinterpret_cast<const float*>(film.p[l]) + H;
      rc = Fb.alloc((size_t)KB * H * sizeof(float));
      if (!rc) rc = launch_pack_vertical(fbeta, L, 0, S, H, 2 * H, Fb.f(), H, 0, st);
      if (rc) return rc;
      GemmEpilogue raw;
      raw.finalize = 0;
      rc = node_gemm(T.f(), KB, Fb.f(), H, out, H, V, H, KB, raw, path, st);
      if (rc) return rc;
    }
    // the target-state operand [coeff(v,l) h_v]: the beta operand is it only for fstride 0 without normalisation (the
    // beta operand uses the raw count)
    if (use_target && (normalize || fstride)) {
      rc = launch_target_term(h_tgt, D, b->row_ptr, V, L, D, normalize, T.f(), K, 0, st);
      if (rc) return rc;
    }
    // gamma for all types in ONE wide contraction: Gall [V, L*H] = h_v [Fgamma_0 | .. | Fgamma_{L-1}] (128-column tiles:
    // the k-block rate of the GEMM pipeline is latency-bound, so work per k-block ~ tile width; 6 GEMMs of N = 320 ran in
    // 80-column tiles at 4.7 ms each, the wide one takes about half of their sum).  Per-type inputs: one GEMM per type,
    // z_l Fgamma_l into columns [l*H, (l+1)*H).
    const int LHw = L * H;
    PoolBuffer Gall{st};
    rc = Gall.alloc((size_t)V * LHw * sizeof(float));
    if (rc) return rc;
    if (fstride == 0) {
      PoolBuffer Fg{st};
      rc = Fg.alloc((size_t)S * LHw * sizeof(float));
      if (!rc) rc = launch_pack_horizontal(film, L, 0, S, H, 2 * H, Fg.f(), LHw, st);   // first H columns of every F_l [S, 2H]
      if (!rc) rc = node_gemm(fin, ldf, Fg.f(), LHw, Gall.f(), LHw, V, LHw, S, none, path, st);
      if (rc) return rc;
    } else {
      for (int l = 0; l < L && !rc; ++l)
        rc = node_gemm(fin + (size_t)l * fstride, ldf, reinterpret_cast<const float*>(film.p[l]), 2 * H,
                       Gall.f() + (size_t)l * H, LHw, V, H, S, none, path, st);
      if (rc) return rc;
    }
    for (int l = 0; l < L; ++l) {
      GemmEpilogue chain;
      chain.mul = Gall.f() + (size_t)l * H; chain.ldm = LHw;
      chain.accumulate = 1;
      chain.finalize = 0;
      const bool last_src = !use_target && l == L - 1;
      if (last_src) {
        chain.finalize = 1;
        chain.act = activation;
        chain.row_norm = agg_row_norm(aggregation); chain.row_ptr = b->row_ptr; chain.V = V; chain.L = L;
      }
      rc = node_gemm(A.f() + (size_t)l * D, K, reinterpret_cast<const float*>(first.p[l]), H, out, H, V, H, D, chain,
                     path, st);
      if (rc) return rc;
      if (use_target) {
        if (l == L - 1) {
          chain.finalize = 1;
          chain.act = activation;
          chain.row_norm = agg_row_norm(aggregation); chain.row_ptr = b->row_ptr; chain.V = V; chain.L = L;
        }
        rc = node_gemm(T.f() + (size_t)l * D, K, reinterpret_cast<const float*>(first.p[l]) + (size_t)D * H, H, out, H, V,
                       H, D, chain, path, st);
        if (rc) return rc;
      }
    }
    return 0;
  }
  // FiLM parameters [gamma_l | beta_l] = z_l F_l depend on (target, type) only (gnn_film.py:99-103); z_l = h_v for
  // fstride 0 (one wide GEMM), else type l's block of fin (one GEMM per type)
  PoolBuffer FB{st};
  auto film_parameters = [&]() {
    int r = FB.alloc((size_t)V * 2 * LH * sizeof(float));
    if (r) return r;
    if (fstride) {
      for (int l = 0; l < L && !r; ++l)
        r = node_gemm(fin + (size_t)l * fstride, ldf, reinterpret_cast<const float*>(film.p[l]), 2 * H,
                      FB.f() + (size_t)l * 2 * H, 2 * LH, V, 2 * H, S, none, path, st);
      return r;
    }
    PoolBuffer Fcat{st};
    r = Fcat.alloc((size_t)S * 2 * LH * sizeof(float));
    if (!r) r = launch_pack_horizontal(film, L, 0, S, 2 * H, 2 * H, Fcat.f(), 2 * LH, st);
    return r ? r : node_gemm(fin, ldf, Fcat.f(), 2 * LH, FB.f(), 2 * LH, V, 2 * LH, S, none, path, st);
  };
  if (num_hidden_layers > 0) {
    // hidden layers in the edge MLP: FiLM parameters at node level, messages on the literal per-edge path
    rc = film_parameters();
    return rc ? rc : edge_mlp_literal(b, h, D, mlp_weights, num_hidden_layers, H, flags, aggregation, activation, FB.f(),
                                      2 * LH, path, out, H, st);
  }
  // projected source messages P_l = h W^s_l  (gnn_edge_mlp.py:100 hoisted to node level)
  PoolBuffer P{st}, Tt{st};
  {
    PoolBuffer Wcat{st};
    rc = P.alloc((size_t)Vs * LH * sizeof(float));
    if (!rc) rc = Wcat.alloc((size_t)D * LH * sizeof(float));
    if (!rc) rc = launch_pack_horizontal(first, L, 0, D, H, H, Wcat.f(), LH, st);
    if (!rc) rc = node_gemm(h, D, Wcat.f(), LH, P.f(), LH, Vs, LH, D, none, path, st);
    if (rc) return rc;
    if (use_target) {
      rc = Tt.alloc((size_t)V * LH * sizeof(float));
      if (!rc) rc = launch_pack_horizontal(first, L, D, D, H, H, Wcat.f(), LH, st);
      if (!rc) rc = node_gemm(h_tgt, D, Wcat.f(), LH, Tt.f(), LH, V, LH, D, none, path, st);
      if (rc) return rc;
    }
  }
  rc = film_parameters();
  if (rc) return rc;
  EdgeReduceParams p;
  p.X = P.f(); p.ldx = LH; p.x_type_stride = H;
  p.T = Tt.f(); p.ldt = LH; p.t_type_stride = H;
  p.G = FB.f(); p.ldg = 2 * LH; p.g_type_stride = 2 * H; p.beta_off = H;
  p.row_ptr = b->row_ptr; p.src = b->src_sorted;
  p.out = out; p.ldo = H; p.V = V; p.L = L; p.C = H;
  p.normalize = normalize;
  p.edge_act = act_before ? activation : TFGNN_ACT_NONE;
  p.reduce_max = aggregation == TFGNN_AGG_MAX;
  p.row_norm = agg_row_norm(aggregation);
  p.final_act = act_before ? TFGNN_ACT_NONE : activation;
  return launch_edge_reduce(p, /*merged=*/true, st);
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_film_fwd(tfgnn_batch_t* b, const float* h, int32_t D, const float* const* mlp_weights,
                                   int32_t num_hidden_layers, const float* const* film_weights, int32_t H,
                                   uint32_t flags, int32_t aggregation, int32_t activation, int32_t path,
                                   float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  TFGNN_REQUIRE(D > 0 && H > 0, "D and H must be positive");
  TFGNN_REQUIRE(valid_act(activation) && valid_agg(aggregation), "unknown activation / aggregation code");
  const float* h_tgt = h ? h + (size_t)b->tgt_off * D : nullptr;
  return film_fwd_core(b, h, D, mlp_weights, num_hidden_layers, h_tgt, 0, D, film_weights, H,
                       flags, aggregation, activation, path, out, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_film_in_fwd(tfgnn_batch_t* b, const float* h, int32_t D, const float* const* mlp_weights,
                                      int32_t num_hidden_layers, const float* film_in, int32_t S,
                                      const float* const* film_weights, int32_t H, uint32_t flags, int32_t aggregation,
                                      int32_t activation, int32_t path, float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "film_in_fwd: batch is NULL");
  TFGNN_REQUIRE(D > 0 && H > 0 && S > 0, "film_in_fwd: D, H and S must be positive");
  TFGNN_REQUIRE(valid_act(activation) && valid_agg(aggregation), "film_in_fwd: unknown activation / aggregation code");
  TFGNN_REQUIRE(film_in || b->V == 0 || b->L == 0, "film_in_fwd: film_in is NULL");
  return film_fwd_core(b, h, D, mlp_weights, num_hidden_layers, film_in, S, S, film_weights, H, flags,
                       aggregation, activation, path, out, (cudaStream_t)stream);
}

namespace tfgnn {

// Node-level attention score halves (rgat.py:111-121 split by linearity of the einsum):
//   s_src[v,l,k] = a_l[k,:d] . P_l[v,k,:]      s_tgt[v,l,k] = a_l[k,d:] . P_l[v,k,:]
// so the per-edge score is leaky_relu(s_src[src] + s_tgt[tgt]).
__global__ void rgat_scores_kernel(const float* __restrict__ P, long long V, int L, int K, int d, PtrTable att,
                                   float* __restrict__ s_src, float* __restrict__ s_tgt) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = V * L * K;
  if (idx >= total) return;
  const int k = (int)(idx % K);
  const int l = (int)((idx / K) % L);
  const long long v = idx / ((long long)K * L);
  const float* a = reinterpret_cast<const float*>(att.p[l]) + (long long)k * 2 * d;
  const float* p = P + v * (long long)(L * K * d) + (long long)l * K * d + (long long)k * d;
  float ss = 0.f, st = 0.f;
  if ((d & 3) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    // 16-byte loads: consecutive threads own consecutive (v,l,k) segments of d floats, so a warp walks one contiguous
    // 32*d-float span and every fetched line is used completely through L1 (the scalar loop ran at 0.6 TB/s: ncu r2c)
    for (int i = 0; i < d; i += 4) {
      const float4 x = ldg_f4(p + i);
      ss = fmaf(a[i], x.x, ss); ss = fmaf(a[i + 1], x.y, ss); ss = fmaf(a[i + 2], x.z, ss); ss = fmaf(a[i + 3], x.w, ss);
      st = fmaf(a[d + i], x.x, st); st = fmaf(a[d + i + 1], x.y, st);
      st = fmaf(a[d + i + 2], x.z, st); st = fmaf(a[d + i + 3], x.w, st);
    }
  } else {
    for (int i = 0; i < d; ++i) {
      const float x = p[i];
      ss = fmaf(a[i], x, ss);
      st = fmaf(a[d + i], x, st);
    }
  }
  s_src[idx] = ss;
  s_tgt[idx] = st;
}

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : kLeakyReluAlpha * x; }

// One thread per (target v, output column c): segment softmax over ALL incoming edges of v (all
// types jointly, rgat.py:135-151) for head k = c/d, then the weighted sum of P_l[src, c].
// Two passes over the node's CSR segments: running max, then exp-sum and weighted accumulate.
// The path of the shapes the target walk (rgat.cu) does not take: d % 4 != 0, L == 0 or an unaligned out.
__global__ void rgat_aggregate_kernel(const float* __restrict__ P, const float* __restrict__ s_src,
                                      const float* __restrict__ s_tgt, const int* __restrict__ row_ptr,
                                      const int* __restrict__ src, long long V, long long tgt_off, int L, int K,
                                      int d, int act, float* __restrict__ out) {
  const int H = K * d;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= V * H) return;
  const long long v = idx / H;
  const int c = (int)(idx % H);
  const int k = c / d;
  const long long LK = (long long)L * K, LH = (long long)L * H;
  float m = kLowestFloat;
  for (int l = 0; l < L; ++l) {
    const long long seg = (long long)l * V + v;
    const int beg = __ldg(row_ptr + seg), end = __ldg(row_ptr + seg + 1);
    const float st = __ldg(s_tgt + (v + tgt_off) * LK + l * K + k);
    for (int e = beg; e < end; ++e)
      m = fmaxf(m, leaky(__ldg(s_src + (long long)__ldg(src + e) * LK + l * K + k) + st));
  }
  float den = 0.f, acc = 0.f;
  for (int l = 0; l < L; ++l) {
    const long long seg = (long long)l * V + v;
    const int beg = __ldg(row_ptr + seg), end = __ldg(row_ptr + seg + 1);
    const float st = __ldg(s_tgt + (v + tgt_off) * LK + l * K + k);
    for (int e = beg; e < end; ++e) {
      const long long u = __ldg(src + e);
      const float w = expf(leaky(__ldg(s_src + u * LK + l * K + k) + st) - m);
      den += w;
      acc = fmaf(w, __ldg(P + u * LH + (long long)l * H + c), acc);
    }
  }
  const float inv = den > 0.f ? 1.0f / den : 0.f;
  out[v * H + c] = apply_act(acc * inv, act);
}

// P_l = h W_l for every one of the Vs nodes and the score halves s_src, s_tgt [Vs, L*K], into the caller's buffers.  The
// forward and the backward (which recomputes them) both call this, so the backward sees the forward's bits.  Needs L > 0.
int rgat_tables(tfgnn_batch* b, const float* h, int D, const PtrTable& wt, const PtrTable& at, int H, int K, int path,
                PoolBuffer& P, PoolBuffer& ss, PoolBuffer& stt, cudaStream_t st) {
  const long long Vs = b->V_src;
  const int L = b->L, d = H / K, LH = L * H;
  PoolBuffer Wcat{st};
  int rc = P.alloc((size_t)Vs * LH * sizeof(float));
  if (!rc) rc = Wcat.alloc((size_t)D * LH * sizeof(float));
  if (!rc) rc = ss.alloc((size_t)Vs * L * K * sizeof(float));
  if (!rc) rc = stt.alloc((size_t)Vs * L * K * sizeof(float));
  // P_l = h W_l for every node once (rgat.py:102-109 applies the same Dense to source and target rows)
  if (!rc) rc = launch_pack_horizontal(wt, L, 0, D, H, H, Wcat.f(), LH, st);
  if (rc) return rc;
  GemmEpilogue none;
  // Attention score halves in the projection's epilogue when the tensor-core GEMM takes the shape and its column tiles hold
  // whole heads (TFGNN_B200_RGAT_FUSED_SCORES=0: separate kernel; read per call, the tests compare the two)
  const char* fs = getenv("TFGNN_B200_RGAT_FUSED_SCORES");
  const bool tc_path = (path == TFGNN_PATH_AUTO || path == TFGNN_PATH_SORTED_TC || path == TFGNN_PATH_FUSED_TC);
  const bool fuse_scores = !(fs && atoi(fs) == 0) && tc_path && gemm_tc_supported(Vs, LH, D, h, D, P.f(), LH) &&
                           gemm_tc_scores_supported(LH, H, d);
  if (fuse_scores) {
    none.score_src = ss.f(); none.score_tgt = stt.f(); none.score_att = at;
    none.score_H = H; none.score_K = K; none.score_d = d;
  }
  rc = node_gemm(h, D, Wcat.f(), LH, P.f(), LH, Vs, LH, D, none, path, st);
  if (rc) return rc;
  if (!fuse_scores) {
    const long long total = Vs * L * K;
    rgat_scores_kernel<<<ceil_div(total, 256), 256, 0, st>>>(P.f(), Vs, L, K, d, at, ss.f(), stt.f());
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_rgat_fwd(tfgnn_batch_t* b, const float* h, int32_t D, const float* const* W,
                                   const float* const* attention, int32_t H, int32_t num_heads,
                                   int32_t activation, int32_t path, float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  TFGNN_REQUIRE(D > 0 && H > 0 && num_heads > 0, "D, H and num_heads must be positive");
  TFGNN_REQUIRE(H % num_heads == 0, "hidden_dim must be divisible by num_heads (rgat.py:72)");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  const long long V = b->V;
  const int L = b->L, K = num_heads, d = H / num_heads;
  if (V == 0) return 0;
  TFGNN_REQUIRE(h && out, "h / out is NULL");
  if (path == TFGNN_PATH_ATOMIC) return unsupported("TFGNN_PATH_ATOMIC is not available for RGAT");
  cudaStream_t st = (cudaStream_t)stream;
  PtrTable wt{}, at{};
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(W && attention && W[l] && attention[l], "a weight pointer is NULL");
    wt.p[l] = W[l];
    at.p[l] = attention[l];
  }
  int rc = batch_enter(b, st);
  if (rc) return rc;
  PoolBuffer P{st}, ss{st}, stt{st};
  if (L > 0) {
    rc = rgat_tables(b, h, D, wt, at, H, K, path, P, ss, stt, st);
    if (rc) return rc;
  }
  const bool vec = (d % 4 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0) && L > 0;
  if (vec) return launch_rgat_aggregate(b, P.f(), ss.f(), stt.f(), K, d, activation, out, st);
  const long long threads = V * H;
  rgat_aggregate_kernel<<<ceil_div(threads, 128), 128, 0, st>>>(
      P.f(), ss.f(), stt.f(), b->row_ptr, b->src_sorted, V, b->tgt_off, L, K, d, activation, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}
