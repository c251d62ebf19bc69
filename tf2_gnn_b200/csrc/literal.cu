// The literal per-edge path: the reference's own op order (message_passing.py:181-218, 165-179) for the
// hyper-parameter combinations whose per-edge non-linearity cannot be hoisted to node level
// (edge MLP with >= 2 hidden layers, or hidden layers combined with max-aggregation /
// activation-before-aggregation / FiLM).  Per edge type, in CSR order (edges of one target contiguous):
//   gather [h_src || h_tgt] -> MLP chain (node_gemm over E_l rows) -> 1/(c+eps), FiLM, activation
//   -> segmented reduce of contiguous rows (no atomics) -> accumulate over types -> row-norm, activation.
// Correctness fallback, not a roofline kernel: it materialises [E_l, max(D_in, H)] twice per type.
#include "layers.cuh"

namespace tfgnn {

// target id of every CSR position of one edge type (positions relative to the type's first edge)
__global__ void expand_targets_kernel(const int* __restrict__ row_ptr, long long V, int l, int* __restrict__ tgt_of) {
  const int base = row_ptr[(long long)l * V];
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    const long long s = (long long)l * V + v;
    for (int e = row_ptr[s]; e < row_ptr[s + 1]; ++e) tgt_of[e - base] = (int)v;
  }
}

// X[e] = [h[src_e] || h_tgt[tgt_e]] : one warp per edge row (tf.nn.embedding_lookup x2 + concat)
__global__ void gather_concat_kernel(const float* __restrict__ h, const float* __restrict__ h_tgt, int D,
                                     const int* __restrict__ row_ptr, const int* __restrict__ src, long long V, int l,
                                     const int* __restrict__ tgt_of, int use_target, float* __restrict__ X, int ldx) {
  const int base = row_ptr[(long long)l * V];
  const int count = row_ptr[(long long)(l + 1) * V] - base;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long e = warp; e < count; e += nwarps) {
    const float* s = h + (long long)src[base + e] * D;
    float* x = X + e * ldx;
    for (int c = lane; c < D; c += 32) x[c] = __ldg(s + c);
    if (use_target) {
      const float* t = h_tgt + (long long)tgt_of[e] * D;
      for (int c = lane; c < D; c += 32) x[D + c] = __ldg(t + c);
    }
  }
}

// per-edge epilogue of the message: scale, FiLM, activation-before-aggregation (in place)
__global__ void edge_post_kernel(float* __restrict__ msg, int H, const int* __restrict__ row_ptr, long long V, int l,
                                 const int* __restrict__ tgt_of, int normalize, const float* __restrict__ FB, int ldf,
                                 int edge_act) {
  const int base = row_ptr[(long long)l * V];
  const long long total = (long long)(row_ptr[(long long)(l + 1) * V] - base) * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i / H;
    const int c = (int)(i - e * H);
    const int v = tgt_of[e];
    float x = msg[i];
    if (normalize) {
      const long long s = (long long)l * V + v;
      x = (1.0f / ((float)(row_ptr[s + 1] - row_ptr[s]) + kSmallNumber)) * x;
    }
    if (FB) {
      const float* f = FB + (long long)v * ldf + (long long)l * 2 * H;
      x = f[c] * x + f[H + c];
    }
    msg[i] = apply_act(x, edge_act);
  }
}

// out[v] = op(out[v], reduce of the contiguous message rows of segment (l, v)); one thread per (v, c)
__global__ void segment_reduce_sorted_kernel(const float* __restrict__ msg, int H, const int* __restrict__ row_ptr,
                                             long long V, int l, int use_max, float* __restrict__ out, int ldo) {
  const int base = row_ptr[(long long)l * V];
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    const int c = (int)(i - v * H);
    const long long s = (long long)l * V + v;
    float acc = out[v * ldo + c];
    for (int e = row_ptr[s]; e < row_ptr[s + 1]; ++e) {
      const float x = msg[(long long)(e - base) * H + c];
      acc = use_max ? fmaxf(acc, x) : acc + x;
    }
    out[v * ldo + c] = acc;
  }
}

__global__ void fill2d_kernel(float* __restrict__ out, long long V, int H, int ldo, float val) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x)
    out[(i / H) * ldo + (i % H)] = val;
}

__global__ void finalize_kernel(float* __restrict__ out, long long V, int H, int ldo, const int* __restrict__ row_ptr,
                                int L, int row_norm, int act) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    float x = out[v * ldo + (i % H)];
    if (row_norm) {
      int cnt = 0;
      for (int l = 0; l < L; ++l) cnt += row_ptr[(long long)l * V + v + 1] - row_ptr[(long long)l * V + v];
      const float n = (float)max(cnt, 1);
      x = x / (row_norm == 1 ? n : sqrtf(n));
    }
    out[v * ldo + (i % H)] = apply_act(x, act);
  }
}

int edge_mlp_literal(tfgnn_batch* b, const float* h, int D, const float* const* mlp_weights, int n_hidden, int H,
                     uint32_t flags, int aggregation, int activation, const float* FB, int ldf, int path, float* out,
                     int ldo, cudaStream_t st) {
  const long long V = b->V;
  const int L = b->L;
  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const bool act_before = flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;
  const bool use_max = aggregation == TFGNN_AGG_MAX;
  const float* h_tgt = h + (size_t)b->tgt_off * D;
  const int D_in = use_target ? 2 * D : D;
  const int n_layers = n_hidden + 1;
  if (path == TFGNN_PATH_ATOMIC) return unsupported("TFGNN_PATH_ATOMIC is not available on the literal per-edge path");
  long long maxE = 1;
  for (int l = 0; l < L; ++l) maxE = b->E[l] > maxE ? b->E[l] : maxE;
  const int wide = D_in > H ? D_in : H;
  int rc = batch_enter(b, st);
  if (rc) return rc;
  PoolBuffer X0{st}, X1{st}, tgt_buf{st};
  rc = X0.alloc((size_t)maxE * wide * sizeof(float));
  if (!rc) rc = X1.alloc((size_t)maxE * wide * sizeof(float));
  if (!rc) rc = tgt_buf.alloc((size_t)maxE * sizeof(int));
  if (rc) return rc;
  const int* tgt_of = (const int*)tgt_buf.p;
  fill2d_kernel<<<grid_for(V * H), 256, 0, st>>>(out, V, H, ldo, use_max ? kLowestFloat : 0.f);
  TFGNN_LAUNCH_CHECK();
  for (int l = 0; l < L; ++l) {
    const long long E = b->E[l];
    if (E == 0) continue;
    expand_targets_kernel<<<grid_for(V), 256, 0, st>>>(b->row_ptr, V, l, (int*)tgt_buf.p);
    TFGNN_LAUNCH_CHECK();
    gather_concat_kernel<<<grid_for(E * 32), 256, 0, st>>>(h, h_tgt, D, b->row_ptr, b->src_sorted, V, l, tgt_of,
                                                         use_target, X0.f(), D_in);
    TFGNN_LAUNCH_CHECK();
    float* cur = X0.f();
    float* nxt = X1.f();
    int k_in = D_in;
    for (int i = 0; i < n_layers; ++i) {
      GemmEpilogue epi;
      epi.act = i < n_hidden ? TFGNN_ACT_RELU : TFGNN_ACT_NONE;   // dpu_utils MLP: ReLU hidden, linear output
      rc = node_gemm(cur, k_in, mlp_weights[l * n_layers + i], H, nxt, H, E, H, k_in, epi, path, st);
      if (rc) return rc;
      float* t = cur; cur = nxt; nxt = t;
      k_in = H;
    }
    edge_post_kernel<<<grid_for(E * H), 256, 0, st>>>(cur, H, b->row_ptr, V, l, tgt_of, normalize, FB, ldf,
                                                     act_before ? activation : TFGNN_ACT_NONE);
    TFGNN_LAUNCH_CHECK();
    segment_reduce_sorted_kernel<<<grid_for(V * H), 256, 0, st>>>(cur, H, b->row_ptr, V, l, use_max, out, ldo);
    TFGNN_LAUNCH_CHECK();
  }
  finalize_kernel<<<grid_for(V * H), 256, 0, st>>>(out, V, H, ldo, b->row_ptr, L, agg_row_norm(aggregation),
                                                  act_before ? TFGNN_ACT_NONE : activation);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn
