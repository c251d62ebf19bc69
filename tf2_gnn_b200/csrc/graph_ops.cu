// Graph-level readout and global exchange (SURVEY.md §8f-4): the segment primitives keyed by node_to_graph_map
// behind WeightedSumGraphRepresentation (nodes_to_graph_representation.py:170-229) and GraphGlobal{Mean,GRU,MLP}Exchange
// (graph_global_exchange.py:83-183).  node_to_graph_map is non-decreasing (graph_dataset.py:211-217; the reference
// itself relies on it: tf.math.segment_sum needs sorted ids), so every graph is a CONTIGUOUS row range and the
// segment reductions need neither atomics nor sorting: graph_ptr[g] .. graph_ptr[g+1].
//
//   graph_offsets           node_to_graph_map -> graph_ptr int32[G+1]
//   segment_softmax         per (graph, head): w = exp((s - max) - log(sum exp(s - max)))   dpu_utils unsorted_segment_softmax
//   weighted_segment_sum    out[g, k*d + c] = sum_{v in g} w[v,k] * r[v, k*d + c]   (or plain sum / mean)
//   gathered_add            out[v] = act((a[v] + b[index[v]]) * scale)              exchange combine (mean, MLP hidden)
//   dense_bias_fwd          Dense with bias (readout MLPs with use_biases, GRU cell halves)
// All HBM-bound and tiny next to the message-passing layers; deterministic (fixed reduction orders).
#include "layers.cuh"

namespace tfgnn {

__global__ void graph_offsets_kernel(const int* __restrict__ n2g, long long V, int G, int* __restrict__ graph_ptr,
                                     int* __restrict__ bad) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= V;
       v += (long long)gridDim.x * blockDim.x) {
    // graphs (prev, cur] start at row v; v == V closes the trailing (possibly empty) graphs
    const int prev = v == 0 ? -1 : __ldg(n2g + v - 1);
    const int cur = v == V ? G : __ldg(n2g + v);
    if (v < V && (cur < prev || cur < 0 || cur >= G)) { atomicAdd(bad, 1); continue; }
    for (int g = prev + 1; g <= cur && g <= G; ++g) graph_ptr[g] = (int)v;
  }
}

// one warp per graph; heads looped.  Two passes over the graph's rows of scores [V, K].
__global__ void segment_softmax_kernel(const float* __restrict__ scores, const int* __restrict__ graph_ptr, int G,
                                       int K, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = warp; g < G; g += nwarps) {
    const int beg = graph_ptr[g], end = graph_ptr[g + 1];
    for (int k = 0; k < K; ++k) {
      float m = kLowestFloat;
      for (int v = beg + lane; v < end; v += 32) m = fmaxf(m, __ldg(scores + (long long)v * K + k));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      float s = 0.f;
      for (int v = beg + lane; v < end; v += 32) s += expf(__ldg(scores + (long long)v * K + k) - m);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float ls = logf(s);
      for (int v = beg + lane; v < end; v += 32)
        out[(long long)v * K + k] = expf((__ldg(scores + (long long)v * K + k) - m) - ls);
    }
  }
}

// CTA = 128 column threads x 4 node lanes; grid = (G, ceil(GD/128)).  Node lane j sums rows beg+j, beg+j+4, ...;
// the four partials are added in lane order (deterministic).
constexpr int kWsCols = 128, kWsLanes = 4;
__global__ void __launch_bounds__(kWsCols * kWsLanes)
weighted_segment_sum_kernel(const float* __restrict__ reprs, const float* __restrict__ weights,
                            const int* __restrict__ graph_ptr, int GD, int K, int mean, float* __restrict__ out) {
  __shared__ float part[kWsLanes][kWsCols];
  const int g = blockIdx.x;
  const int c = blockIdx.y * kWsCols + threadIdx.x;
  const int j = threadIdx.y;
  const int beg = graph_ptr[g], end = graph_ptr[g + 1];
  const int d = GD / K;
  float acc = 0.f;
  if (c < GD) {
    const int k = c / d;
    for (int v = beg + j; v < end; v += kWsLanes) {
      const float r = __ldg(reprs + (long long)v * GD + c);
      acc += weights ? __ldg(weights + (long long)v * K + k) * r : r;
    }
  }
  part[j][threadIdx.x] = acc;
  __syncthreads();
  if (j == 0 && c < GD) {
    float s = part[0][threadIdx.x];
#pragma unroll
    for (int t = 1; t < kWsLanes; ++t) s += part[t][threadIdx.x];
    if (mean) s = s / (float)max(end - beg, 1);
    out[(long long)g * GD + c] = s;
  }
}

__global__ void gathered_add_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                    const int* __restrict__ index, long long V, int H, float scale, int act,
                                    float* __restrict__ out) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    const int c = (int)(i - v * H);
    const long long r = index ? (long long)__ldg(index + v) : v;
    out[i] = apply_act((a[i] + __ldg(b + r * H + c)) * scale, act);
  }
}

__global__ void clamp_kernel(float* __restrict__ x, long long n, float lo, float hi, int has_lo, int has_hi) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (has_lo) v = fmaxf(v, lo);
    if (has_hi) v = fminf(v, hi);
    x[i] = v;
  }
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_graph_offsets(const int32_t* node_to_graph_map, int64_t num_nodes, int32_t num_graphs,
                                        int32_t* graph_ptr, int32_t validate, void* stream) {
  TFGNN_REQUIRE(num_nodes >= 0 && num_nodes < (1ll << 31) && num_graphs >= 0, "bad graph_offsets sizes");
  TFGNN_REQUIRE(graph_ptr != nullptr, "graph_ptr is NULL");
  TFGNN_REQUIRE(num_nodes == 0 || node_to_graph_map != nullptr, "node_to_graph_map is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer bad_buf{st};
  int rc = bad_buf.alloc(sizeof(int));
  if (rc) return rc;
  int* bad = (int*)bad_buf.p;
  TFGNN_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
  graph_offsets_kernel<<<grid_for(num_nodes + 1), 256, 0, st>>>(node_to_graph_map, num_nodes, num_graphs, graph_ptr, bad);
  TFGNN_LAUNCH_CHECK();
  int host_bad = 0;
  if (validate) {
    TFGNN_CUDA(cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    TFGNN_CUDA(cudaStreamSynchronize(st));
  }
  if (host_bad) {
    set_error(TFGNN_ERR_INVALID_ARGUMENT,
              "node_to_graph_map must be non-decreasing with values in [0, num_graphs) (graph_dataset.py:211-217)");
    return TFGNN_ERR_INVALID_ARGUMENT;
  }
  return 0;
}

extern "C" int tfgnn_b200_segment_softmax(const float* scores, const int32_t* graph_ptr, int32_t num_graphs,
                                          int32_t num_heads, float* out, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0 && num_heads > 0, "bad segment_softmax sizes");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(scores && graph_ptr && out, "NULL pointer");
  int blocks = ceil_div((long long)num_graphs * 32, 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  segment_softmax_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(scores, graph_ptr, num_graphs, num_heads, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_weighted_segment_sum(const float* node_reprs, const float* weights, const int32_t* graph_ptr,
                                               int32_t num_graphs, int32_t repr_dim, int32_t num_heads, int32_t mean,
                                               float* out, void* stream) {
  TFGNN_REQUIRE(num_graphs >= 0 && repr_dim > 0 && num_heads > 0 && repr_dim % num_heads == 0,
                "bad weighted_segment_sum sizes (num_heads must divide the representation size)");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(node_reprs && graph_ptr && out, "NULL pointer");
  dim3 grid((unsigned)num_graphs, (unsigned)((repr_dim + kWsCols - 1) / kWsCols));
  dim3 block(kWsCols, kWsLanes);
  weighted_segment_sum_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(node_reprs, weights, graph_ptr, repr_dim,
                                                                        num_heads, mean, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_gathered_add(const float* a, const float* b, const int32_t* index, int64_t num_rows,
                                       int32_t H, float scale, int32_t activation, float* out, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && H > 0 && valid_act(activation), "bad gathered_add arguments");
  if (num_rows == 0) return 0;
  TFGNN_REQUIRE(a && b && out, "NULL pointer");
  gathered_add_kernel<<<grid_for(num_rows * H), 256, 0, (cudaStream_t)stream>>>(a, b, index, num_rows, H, scale,
                                                                              activation, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_clamp(float* x, int64_t n, float lower, float upper, int32_t has_lower, int32_t has_upper,
                                void* stream) {
  TFGNN_REQUIRE(n >= 0, "negative size");
  if (n == 0 || (!has_lower && !has_upper)) return 0;
  TFGNN_REQUIRE(x != nullptr, "NULL pointer");
  clamp_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, n, lower, upper, has_lower, has_upper);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_dense_bias_fwd(const float* x, const float* W, const float* bias, float* out, int64_t V,
                                         int32_t K, int32_t N, int32_t activation, int32_t path, void* stream) {
  TFGNN_REQUIRE(V >= 0 && K > 0 && N > 0, "bad dense shape");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  if (V == 0) return 0;
  TFGNN_REQUIRE(x && W && out, "NULL pointer");
  GemmEpilogue epi;
  epi.act = activation;
  epi.bias = bias;
  return node_gemm(x, K, W, N, out, N, V, N, K, epi, path, (cudaStream_t)stream);
}
