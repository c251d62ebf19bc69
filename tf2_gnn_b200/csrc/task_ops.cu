// Task losses and metrics of tf2_gnn.models (SURVEY.md row 13): the node multiclass loss with its micro-F1 counts
// (node_multiclass_task.py:57-70), the graph regression MSE / MAE (graph_regression_task.py:152-166) and the graph binary
// cross-entropy with its number of correct predictions (graph_binary_classification_task.py:33-58).
//
//   *_fwd   one pass over the table: each CTA reduces one fixed chunk of kLossChunk elements (row-major, so whole rows in
//           row order) into one partial per sum, then one CTA combines the partials in chunk order and writes the
//           scalars.  The result is a function of the inputs alone (not of the grid); counts are exact int64.
//   *_bwd   elementwise; the upstream scalar gradient is read from device memory, so a training step never waits on
//           the host.
#include <math.h>

#include "layers.cuh"

namespace tfgnn {

constexpr int kLossThreads = 256;
constexpr int kLossChunk = 4096;   // elements per partial (a constant: the sums must not depend on the grid)

// Sums of NF floats and NI counts over a CTA, in a fixed tree order.  Thread 0 holds the result.
template <int NF, int NI>
__device__ __forceinline__ void cta_sum(float (&f)[NF], long long (&c)[NI]) {
  __shared__ float sf[NF > 0 ? NF : 1][kLossThreads];
  __shared__ long long sc[NI > 0 ? NI : 1][kLossThreads];
#pragma unroll
  for (int k = 0; k < NF; ++k) sf[k][threadIdx.x] = f[k];
#pragma unroll
  for (int k = 0; k < NI; ++k) sc[k][threadIdx.x] = c[k];
  __syncthreads();
  for (int s = kLossThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int k = 0; k < NF; ++k) sf[k][threadIdx.x] += sf[k][threadIdx.x + s];
#pragma unroll
      for (int k = 0; k < NI; ++k) sc[k][threadIdx.x] += sc[k][threadIdx.x + s];
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < NF; ++k) f[k] = sf[k][0];
#pragma unroll
  for (int k = 0; k < NI; ++k) c[k] = sc[k][0];
}

// where the finish kernel writes: up to two float scalars and the counts (0 / 0 = NaN for an empty batch, as tf.reduce_mean)
struct LossOut {
  float* f0;
  float* f1;
  long long* c;
};

__device__ __forceinline__ float sigmoid_f32(float x) { return 1.f / (1.f + expf(-x)); }

// tf.nn.sigmoid_cross_entropy_with_logits and the micro-F1 counts of one (logit, label) pair.
struct NodeMulticlassOp {
  static constexpr int NF = 1, NI = 3;
  const float* x;
  const float* y;
  __device__ __forceinline__ void add(long long i, float (&f)[NF], long long (&c)[NI]) const {
    const float xi = __ldg(x + i), yi = __ldg(y + i);
    f[0] += fmaxf(xi, 0.f) - xi * yi + log1pf(expf(-fabsf(xi)));
    const int p = (int)rintf(sigmoid_f32(xi));   // tf.math.round: half to even, so a logit of 0 predicts 0
    const int l = (int)yi;
    c[0] += p * l != 0;
    c[1] += p * (l - 1) != 0;
    c[2] += (p - 1) * l != 0;
  }
  // micro_f1 (node_multiclass_task.py:10-23): int64 / int64 is float64 in TF; NaN whenever tp == 0 (0 / 0)
  static __device__ void finish(const float (&f)[NF], const long long (&c)[NI], float n, const LossOut& o) {
    *o.f0 = f[0] / n;
    const double tp = (double)c[0], prec = tp / (tp + (double)c[1]), rec = tp / (tp + (double)c[2]);
    *o.f1 = (float)((2.0 * prec * rec) / (prec + rec));
#pragma unroll
    for (int k = 0; k < NI; ++k) o.c[k] = c[k];
  }
};

struct GraphRegressionOp {
  static constexpr int NF = 2, NI = 0;
  const float* p;
  const float* t;
  __device__ __forceinline__ void add(long long i, float (&f)[NF], long long (&)[NI > 0 ? NI : 1]) const {
    const float d = __ldg(p + i) - __ldg(t + i);
    f[0] += d * d;
    f[1] += fabsf(d);
  }
  static __device__ void finish(const float (&f)[NF], const long long (&)[1], float n, const LossOut& o) {
    *o.f0 = f[0] / n;
    *o.f1 = f[1] / n;
  }
};

// Keras backend.binary_crossentropy(from_logits=False), TF >= 2.2
constexpr float kBceEps = 1e-7f;
struct GraphBinaryOp {
  static constexpr int NF = 1, NI = 1;
  const float* p;
  const float* t;
  __device__ __forceinline__ void add(long long i, float (&f)[NF], long long (&c)[NI]) const {
    const float pi = __ldg(p + i), ti = __ldg(t + i);
    const float q = fminf(fmaxf(pi, kBceEps), 1.f - kBceEps);
    f[0] += ti * logf(q + kBceEps) + (1.f - ti) * logf(1.f - q + kBceEps);
    c[0] += ti == rintf(pi);
  }
  static __device__ void finish(const float (&f)[NF], const long long (&c)[NI], float n, const LossOut& o) {
    *o.f0 = -(f[0] / n);
    o.c[0] = c[0];
  }
};

// grid = chunks; partials: float [chunks][NF], long long [chunks][NI]
template <class Op>
__global__ void __launch_bounds__(kLossThreads)
loss_chunks_kernel(Op op, long long n, float* __restrict__ fpart, long long* __restrict__ cpart) {
  constexpr int NF = Op::NF, NI = Op::NI > 0 ? Op::NI : 1;
  float f[NF];
  long long c[NI];
#pragma unroll
  for (int k = 0; k < NF; ++k) f[k] = 0.f;
#pragma unroll
  for (int k = 0; k < NI; ++k) c[k] = 0;
  const long long beg = (long long)blockIdx.x * kLossChunk;
  const long long end = beg + kLossChunk < n ? beg + kLossChunk : n;
  for (long long i = beg + threadIdx.x; i < end; i += kLossThreads) op.add(i, f, c);
  cta_sum<NF, NI>(f, c);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NF; ++k) fpart[(long long)blockIdx.x * NF + k] = f[k];
    if (Op::NI > 0)
#pragma unroll
      for (int k = 0; k < NI; ++k) cpart[(long long)blockIdx.x * NI + k] = c[k];
  }
}

// One CTA: thread j adds chunks j, j + kLossThreads, ... in order, the threads' sums are combined in a fixed tree, and
// Op::finish turns the sums over n rows into the outputs.
template <class Op>
__global__ void __launch_bounds__(kLossThreads)
loss_finish_kernel(const float* __restrict__ fpart, const long long* __restrict__ cpart, int chunks, float n, LossOut o) {
  constexpr int NF = Op::NF, NI = Op::NI > 0 ? Op::NI : 1;
  float f[NF];
  long long c[NI];
#pragma unroll
  for (int k = 0; k < NF; ++k) f[k] = 0.f;
#pragma unroll
  for (int k = 0; k < NI; ++k) c[k] = 0;
  for (int j = threadIdx.x; j < chunks; j += kLossThreads) {
#pragma unroll
    for (int k = 0; k < NF; ++k) f[k] += fpart[(long long)j * NF + k];
    if (Op::NI > 0)
#pragma unroll
      for (int k = 0; k < NI; ++k) c[k] += cpart[(long long)j * NI + k];
  }
  cta_sum<NF, NI>(f, c);
  if (threadIdx.x == 0) Op::finish(f, c, n, o);
}

template <class Op>
int loss_fwd(const Op& op, long long n, float rows, const LossOut& out, cudaStream_t st) {
  constexpr int NIc = Op::NI > 0 ? Op::NI : 1;
  const int chunks = ceil_div(n, kLossChunk);
  PoolBuffer fpart{st}, cpart{st};
  int rc = fpart.alloc((size_t)chunks * Op::NF * sizeof(float));
  if (!rc) rc = cpart.alloc((size_t)chunks * NIc * sizeof(long long));
  if (rc) return rc;
  if (chunks) {
    loss_chunks_kernel<Op><<<chunks, kLossThreads, 0, st>>>(op, n, fpart.f(), (long long*)cpart.p);
    TFGNN_LAUNCH_CHECK();
  }
  loss_finish_kernel<Op><<<1, kLossThreads, 0, st>>>(fpart.f(), (const long long*)cpart.p, chunks, rows, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// ---- the node loss on target-range shards --------------------------------------------------------------------------
// One CTA, one thread: the ranks' raw sums and counts added left to right in rank order, then the finish of _fwd over
// the batch's total row count.  Every rank that holds the same gathered partials writes the same bits.
__global__ void node_multiclass_merge_kernel(const float* __restrict__ loss_sums, const long long* __restrict__ counts,
                                             int world, float n, LossOut o) {
  if (threadIdx.x != 0) return;
  float f[NodeMulticlassOp::NF] = {loss_sums[0]};
  long long c[NodeMulticlassOp::NI] = {counts[0], counts[1], counts[2]};
  for (int r = 1; r < world; ++r) {
    f[0] += loss_sums[r];
#pragma unroll
    for (int k = 0; k < NodeMulticlassOp::NI; ++k) c[k] += counts[(long long)r * NodeMulticlassOp::NI + k];
  }
  NodeMulticlassOp::finish(f, c, n, o);
}

// ---- backward ----------------------------------------------------------------------------------------------------
// grad = g * (sigmoid(x) - y) / V
__global__ void node_multiclass_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, long long n, float inv_V,
                                           const float* __restrict__ g, float* __restrict__ grad) {
  const float s = __ldg(g) * inv_V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    grad[i] = s * (sigmoid_f32(__ldg(x + i)) - __ldg(y + i));
}

// grad = g * 2 (p - t) / G
__global__ void graph_regression_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t, long long n, float inv_G,
                                            const float* __restrict__ g, float* __restrict__ grad) {
  const float s = 2.f * __ldg(g) * inv_G;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    grad[i] = s * (__ldg(p + i) - __ldg(t + i));
}

// d/dp of -mean[t log(q + eps) + (1 - t) log(1 - q + eps)], q = clip(p, eps, 1 - eps): zero where the clip cut
// (tf.clip_by_value passes the gradient where lo <= p <= hi).
__global__ void graph_binary_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t, long long n, float inv_G,
                                        const float* __restrict__ g, float* __restrict__ grad) {
  const float s = -__ldg(g) * inv_G;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float pi = __ldg(p + i), ti = __ldg(t + i);
    const bool pass = pi >= kBceEps && pi <= 1.f - kBceEps;
    const float q = fminf(fmaxf(pi, kBceEps), 1.f - kBceEps);
    grad[i] = pass ? s * (ti / (q + kBceEps) - (1.f - ti) / (1.f - q + kBceEps)) : 0.f;
  }
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_node_multiclass_loss_fwd(const float* logits, const float* labels, int64_t num_nodes,
                                                   int32_t num_labels, float* loss, float* f1_score, int64_t* f1_counts,
                                                   void* stream) {
  TFGNN_REQUIRE(num_nodes >= 0 && num_labels > 0, "tfgnn_b200_node_multiclass_loss_fwd: bad sizes (num_labels must be > 0)");
  TFGNN_REQUIRE(loss && f1_score && f1_counts && (num_nodes == 0 || (logits && labels)),
                "tfgnn_b200_node_multiclass_loss_fwd: NULL pointer");
  NodeMulticlassOp op{logits, labels};
  return loss_fwd(op, num_nodes * num_labels, (float)num_nodes, LossOut{loss, f1_score, (long long*)f1_counts},
                  (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_node_multiclass_loss_bwd(const float* logits, const float* labels, int64_t num_nodes,
                                                   int32_t num_labels, const float* grad_loss, float* grad_logits,
                                                   void* stream) {
  TFGNN_REQUIRE(num_nodes >= 0 && num_labels > 0, "tfgnn_b200_node_multiclass_loss_bwd: bad sizes (num_labels must be > 0)");
  if (num_nodes == 0) return 0;
  TFGNN_REQUIRE(logits && labels && grad_loss && grad_logits, "tfgnn_b200_node_multiclass_loss_bwd: NULL pointer");
  const long long n = num_nodes * num_labels;
  node_multiclass_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(logits, labels, n, 1.f / (float)num_nodes,
                                                                          grad_loss, grad_logits);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// The pass of _fwd over a rank's rows, finished over one row: f[0] / 1.0f is the raw sum, exactly.
extern "C" int tfgnn_b200_node_multiclass_loss_partial(const float* logits, const float* labels, int64_t num_rows,
                                                       int32_t num_labels, float* loss_sum, int64_t* f1_counts,
                                                       void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && num_labels > 0,
                "tfgnn_b200_node_multiclass_loss_partial: bad sizes (num_labels must be > 0)");
  TFGNN_REQUIRE(loss_sum && f1_counts && (num_rows == 0 || (logits && labels)),
                "tfgnn_b200_node_multiclass_loss_partial: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer unused_f1{st};   // the finish writes an F1 of the rank's counts; only the merged one is meaningful
  int rc = unused_f1.alloc(sizeof(float));
  if (rc) return rc;
  NodeMulticlassOp op{logits, labels};
  return loss_fwd(op, num_rows * num_labels, 1.f, LossOut{loss_sum, unused_f1.f(), (long long*)f1_counts}, st);
}

extern "C" int tfgnn_b200_node_multiclass_loss_merge(const float* loss_sums, const int64_t* counts, int32_t world,
                                                     int64_t total_rows, float* loss, float* f1_score, int64_t* f1_counts,
                                                     void* stream) {
  TFGNN_REQUIRE(world >= 1 && total_rows >= 0,
                "tfgnn_b200_node_multiclass_loss_merge: bad sizes (world must be >= 1, total_rows >= 0)");
  TFGNN_REQUIRE(loss_sums && counts && loss && f1_score && f1_counts, "tfgnn_b200_node_multiclass_loss_merge: NULL pointer");
  node_multiclass_merge_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(
      loss_sums, (const long long*)counts, world, (float)total_rows, LossOut{loss, f1_score, (long long*)f1_counts});
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_node_multiclass_loss_bwd_rows(const float* logits, const float* labels, int64_t num_rows,
                                                        int32_t num_labels, int64_t total_rows, const float* grad_loss,
                                                        float* grad_logits, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && num_labels > 0 && total_rows >= num_rows,
                "tfgnn_b200_node_multiclass_loss_bwd_rows: bad sizes (num_labels must be > 0, total_rows >= num_rows)");
  if (num_rows == 0) return 0;
  TFGNN_REQUIRE(logits && labels && grad_loss && grad_logits, "tfgnn_b200_node_multiclass_loss_bwd_rows: NULL pointer");
  const long long n = num_rows * num_labels;
  node_multiclass_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(logits, labels, n, 1.f / (float)total_rows,
                                                                          grad_loss, grad_logits);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_graph_regression_loss_fwd(const float* pred, const float* target, int64_t num_graphs,
                                                    float* mse, float* mae, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0, "tfgnn_b200_graph_regression_loss_fwd: negative num_graphs");
  TFGNN_REQUIRE(mse && mae && (num_graphs == 0 || (pred && target)), "tfgnn_b200_graph_regression_loss_fwd: NULL pointer");
  GraphRegressionOp op{pred, target};
  return loss_fwd(op, num_graphs, (float)num_graphs, LossOut{mse, mae, nullptr}, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_graph_regression_loss_bwd(const float* pred, const float* target, int64_t num_graphs,
                                                    const float* grad_loss, float* grad_pred, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0, "tfgnn_b200_graph_regression_loss_bwd: negative num_graphs");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(pred && target && grad_loss && grad_pred, "tfgnn_b200_graph_regression_loss_bwd: NULL pointer");
  graph_regression_bwd_kernel<<<grid_for(num_graphs), 256, 0, (cudaStream_t)stream>>>(
      pred, target, num_graphs, 1.f / (float)num_graphs, grad_loss, grad_pred);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_graph_binary_loss_fwd(const float* prob, const float* target, int64_t num_graphs, float* loss,
                                                int64_t* num_correct, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0, "tfgnn_b200_graph_binary_loss_fwd: negative num_graphs");
  TFGNN_REQUIRE(loss && num_correct && (num_graphs == 0 || (prob && target)),
                "tfgnn_b200_graph_binary_loss_fwd: NULL pointer");
  GraphBinaryOp op{prob, target};
  return loss_fwd(op, num_graphs, (float)num_graphs, LossOut{loss, nullptr, (long long*)num_correct}, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_graph_binary_loss_bwd(const float* prob, const float* target, int64_t num_graphs,
                                                const float* grad_loss, float* grad_prob, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0, "tfgnn_b200_graph_binary_loss_bwd: negative num_graphs");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(prob && target && grad_loss && grad_prob, "tfgnn_b200_graph_binary_loss_bwd: NULL pointer");
  graph_binary_bwd_kernel<<<grid_for(num_graphs), 256, 0, (cudaStream_t)stream>>>(prob, target, num_graphs,
                                                                                1.f / (float)num_graphs, grad_loss,
                                                                                grad_prob);
  TFGNN_LAUNCH_CHECK();
  return 0;
}
