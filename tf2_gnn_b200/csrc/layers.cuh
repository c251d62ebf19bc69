#pragma once
#include "common.cuh"
#include "edge_reduce.cuh"
#include "gemm.cuh"

namespace tfgnn {
int unsupported(const std::string& msg);
bool valid_act(int a);
bool valid_agg(int a);
int agg_row_norm(int aggregation);
int node_gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, long long M, int N, int K,
              const GemmEpilogue& epi, int path, cudaStream_t st);
// P, T (into the caller's buffers) and the merged edge reduce of the transform-then-aggregate form (api.cu)
int transform_aggregate_tables(tfgnn_batch* b, const float* h, int D, const PtrTable& W, int H, uint32_t flags,
                               int aggregation, int activation, int path, PoolBuffer& P, PoolBuffer& T,
                               EdgeReduceParams* p, cudaStream_t st);
int edge_mlp_core(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights, int n_hidden, int H,
                  uint32_t flags, int aggregation, int activation, int path, float* out, int ldo, cudaStream_t st);
// GGNN's node update out = GRUCell(agg, h) over V rows (variants.cu): agg [V, H], state rows h [V, ldh], out [V, H];
// in_place: out overlaps the caller's state table (the update then keeps the two GEMMs and the gate kernel)
int gru_update(const float* agg, const float* h, int ldh, const float* gru_kernel, const float* gru_recurrent_kernel,
               const float* gru_bias, long long V, int H, int path, bool in_place, float* out, cudaStream_t st);
// GNN-FiLM forward (variants.cu) with FiLM input rows fin [V, L*S]: type l reads columns [l*fstride, l*fstride + S) through
// film_weights[l] [S, 2H]; fstride 0 with fin = the owned rows of h [V, D] and S = D is tfgnn_b200_film_fwd
int film_fwd_core(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights, int num_hidden_layers,
                  const float* fin, int fstride, int S, const float* const* film_weights, int H, uint32_t flags,
                  int aggregation, int activation, int path, float* out, cudaStream_t st);
// literal per-edge path (literal.cu); FB = optional FiLM table [V, L*2H] (gamma | beta per type)
int edge_mlp_literal(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights, int n_hidden, int H,
                     uint32_t flags, int aggregation, int activation, const float* FB, int ldf, int path, float* out,
                     int ldo, cudaStream_t st);
// RGAT edge-level aggregation (rgat.cu): the target walk in output mode, out = act(o) [V, H]; needs (H/K) % 4 == 0
int launch_rgat_aggregate(tfgnn_batch* b, const float* P, const float* s_src, const float* s_tgt, int K, int d,
                          int activation, float* out, cudaStream_t st);
// RGAT projection P and score halves s_src, s_tgt of the forward, into the caller's buffers (variants.cu); L > 0
int rgat_tables(tfgnn_batch* b, const float* h, int D, const PtrTable& wt, const PtrTable& at, int H, int K, int path,
                PoolBuffer& P, PoolBuffer& s_src, PoolBuffer& s_tgt, cudaStream_t st);
// Edge-level steps of the RGAT backward (rgat.cu), no float atomics; d % 4 == 0, H <= 512.
//   target pass (the target walk in statistics mode): stat [V, 3K] = (m, den, g) per head, ds_tgt [V, L*K]
//   source pass over bt's source-keyed CSR: dP [Vs, L*H], ds_src [Vs, L*K]
//   attention gradient: rows of ds [rows, L*K] and P (ldP = L*H) -> half `half` (0: source, 1: target) of every grad_att[l]
int launch_rgat_target_pass(tfgnn_batch* b, const float* P, const float* s_src, const float* s_tgt, int K, int d,
                            const float* dz, float* stat, float* ds_tgt, cudaStream_t st);
int launch_rgat_source_pass(const tfgnn_batch* b, const tfgnn_batch* bt, const float* P, const float* s_src,
                            const float* s_tgt, const PtrTable& att, int K, int d, const float* dz, const float* stat,
                            const float* ds_tgt, float* dP, float* ds_src, cudaStream_t st);
int launch_rgat_attention_grad(const float* ds, const float* P, long long rows, int L, int K, int d, const PtrTable& grad_att,
                               int half, cudaStream_t st);
}  // namespace tfgnn
