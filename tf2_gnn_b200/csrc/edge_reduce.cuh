#pragma once
#include "common.cuh"

namespace tfgnn {

// Parameters of the edge-level gather/reduce kernels (edge_reduce.cu).
struct EdgeReduceParams {
  const float* X = nullptr;  // node table gathered by source id, [V, ldx]; type l reads columns
  int ldx = 0;               //   [l*x_type_stride, l*x_type_stride + C)
  int x_type_stride = 0;
  const float* T = nullptr;  // optional target-side additive table (same addressing with ldt/t_type_stride)
  int ldt = 0;
  int t_type_stride = 0;
  const float* G = nullptr;  // optional FiLM table: gamma at G[v, l*g_type_stride + c], beta at + beta_off
  int ldg = 0;
  int g_type_stride = 0;
  int beta_off = 0;
  const int* row_ptr = nullptr;
  const int* src = nullptr;
  float* out = nullptr;      // PER_TYPE: out[v, l*out_type_stride + c]; MERGED: out[v, c]
  int ldo = 0;
  int out_type_stride = 0;
  int V = 0, L = 0, C = 0;
  int v_begin = 0, v_count = 0;  // target-node range handled by this launch (v_count 0 = all V);
                                 // output rows are relative to v_begin
  int normalize = 0;    // multiply by 1/(c_{v,l}+1e-7)                        gnn_edge_mlp.py:102-106
  int hidden_relu = 0;  // per-edge ReLU of the (pre-projected) hidden layer   dpu_utils MLP
  int edge_act = 0;     // activation before aggregation                      message_passing.py:169-170
  int reduce_max = 0;   // unsorted_segment_max instead of sum
  int row_norm = 0;     // MERGED only: 1 = mean, 2 = sqrt_n (counts over all types)
  int final_act = 0;    // MERGED only: activation after aggregation          message_passing.py:176-177
  float* ties = nullptr;  // MERGED max only: [v, c] (leading dimension ldo) = number of messages equal to the maximum
};

// max_blocks > 0 caps the grid (grid-stride over segments) so another kernel can co-reside on the SMs.
int launch_edge_reduce(const EdgeReduceParams& p, bool merged, cudaStream_t st, int max_blocks = 0);
// Gradient of the merged transform-then-aggregate reduce f (max and / or activation before aggregation) with respect to its
// per-type tables, for z = its maximum ([V, C]; max only, else NULL) and dz = the gradient of its result ([V, C], the tie
// count of max divided out).  With the source-keyed CSR (row_ptr_t, tgt over Vs sources): dP = d/d f.X into out [Vs, L*C];
// with row_ptr_t NULL: dT = d/d f.T over f's own CSR into out [V, L*C].
int launch_edge_grad(const EdgeReduceParams& f, const float* z, const float* dz, const int* row_ptr_t, const int* tgt,
                     int Vs, float* out, cudaStream_t st);
// out[v, col0 + l*D + c] = coeff(v,l) h[v, l*in_stride + c], coeff = c_{v,l} or c/(c+eps) (normalize); in_stride 0: one
// input row for every type (the target-state term), else one input block per type (GNN-FiLM's per-type FiLM input).
int launch_target_term(const float* h, int ldh, const int* row_ptr, int V, int L, int D, int normalize,
                       float* out, int ldo, int col0, cudaStream_t st, int in_stride = 0);
int launch_edge_scatter_atomic(const tfgnn_batch* b, const float* X, int ldx, int C, int normalize,
                               float* out, int ldo, int type_stride, cudaStream_t st);

}  // namespace tfgnn
