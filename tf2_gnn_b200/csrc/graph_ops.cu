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
//   segment_sum_rows        out[g] = sum_{v in g} data[v]: adjoint of table[node_to_graph_map], fixed 64-row chunks
//   readout_bwd             gradients of weighted_segment_sum through the weighting and the clamp, one pass over the nodes
//   readout_partial / _merge  the readout of a target-range shard: per-graph (max, sum, weighted sum) partials of the
//                           owned rows, and the rank-ordered online-softmax merge of every rank's partials
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

// ---- backward: segment sum over graph row ranges, readout backward -------------------------------------------------
// segment_sum_rows: the rows are cut into chunks of kSegRows rows (a constant: the result must not depend on the grid).
// One thread per column (float4 of columns when VEC) walks its chunk's rows in row order and emits a value whenever the
// graph changes: a graph that lies inside the chunk is final and goes to `out`; the graph that entered from the previous
// chunk leaves its sum in the chunk's head slot, the graph that continues into the next chunk in the tail slot.
constexpr int kSegRows = 64, kSegThreads = 64, kSegBatch = 8, kSegLanes = 8, kSegCols = 32;

template <bool VEC>
struct SegVal;
template <>
struct SegVal<true> {
  using T = float4;
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ T load(const float* p) { return ldg_f4(p); }
  static __device__ __forceinline__ void add(T& a, const T& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
  static __device__ __forceinline__ void store(float* p, const T& v) { *reinterpret_cast<float4*>(p) = v; }
};
template <>
struct SegVal<false> {
  using T = float;
  static __device__ __forceinline__ T zero() { return 0.f; }
  static __device__ __forceinline__ T load(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void add(T& a, const T& b) { a += b; }
  static __device__ __forceinline__ void store(float* p, const T& v) { *p = v; }
};

// grid = (chunks, column tiles of kSegThreads values); partial [chunks][2][C]
template <bool VEC>
__global__ void __launch_bounds__(kSegThreads)
segment_sum_chunks_kernel(const float* __restrict__ data, const int* __restrict__ n2g,
                          const int* __restrict__ graph_ptr, long long V, int C, float* __restrict__ out,
                          float* __restrict__ partial) {
  using S = SegVal<VEC>;
  constexpr int W = VEC ? 4 : 1;
  __shared__ int row_graph[kSegRows];
  const long long r0 = (long long)blockIdx.x * kSegRows;
  const int rows = (int)(V - r0 < kSegRows ? V - r0 : kSegRows);
  for (int j = threadIdx.x; j < rows; j += kSegThreads) row_graph[j] = __ldg(n2g + r0 + j);
  __syncthreads();
  const int c = (blockIdx.y * kSegThreads + threadIdx.x) * W;
  if (c >= C) return;
  auto emit = [&](int g, const typename S::T& acc) {
    const long long beg = graph_ptr[g], end = graph_ptr[g + 1];
    float* dst = beg < r0 ? partial + ((long long)blockIdx.x * 2) * C
                          : (end > r0 + rows ? partial + ((long long)blockIdx.x * 2 + 1) * C : out + (long long)g * C);
    S::store(dst + c, acc);
  };
  int cur = row_graph[0];
  typename S::T acc = S::zero();
  for (int j0 = 0; j0 < rows; j0 += kSegBatch) {
    typename S::T buf[kSegBatch];
#pragma unroll
    for (int j = 0; j < kSegBatch; ++j)
      if (j0 + j < rows) buf[j] = S::load(data + (r0 + j0 + j) * C + c);
#pragma unroll
    for (int j = 0; j < kSegBatch; ++j) {
      if (j0 + j < rows) {
        const int g = row_graph[j0 + j];
        if (g != cur) {
          emit(cur, acc);
          acc = S::zero();
          cur = g;
        }
        S::add(acc, buf[j]);
      }
    }
  }
  emit(cur, acc);
}

// Graphs that cross a chunk border: the tail slot of their first chunk, then the head slots of the chunks that follow, added
// by kSegLanes lanes (lane j takes items j, j + kSegLanes, ...) whose sums are added in lane order.  Empty graphs get zeros.
// block = (kSegCols, kSegLanes); grid = (graphs, strided; column tiles)
__global__ void __launch_bounds__(kSegCols * kSegLanes)
segment_sum_finish_kernel(const float* __restrict__ partial, const int* __restrict__ graph_ptr, int G, int C,
                          float* __restrict__ out) {
  __shared__ float part[kSegLanes][kSegCols];
  const int c = blockIdx.y * kSegCols + threadIdx.x;
  const int j = threadIdx.y;
  for (int g = blockIdx.x; g < G; g += gridDim.x) {
    const int beg = graph_ptr[g], end = graph_ptr[g + 1];
    if (beg == end) {
      if (j == 0 && c < C) out[(long long)g * C + c] = 0.f;
      continue;
    }
    const int first = beg / kSegRows, last = (end - 1) / kSegRows;
    if (first == last) continue;   // final since the first kernel
    float s = 0.f;
    if (c < C)
      for (int t = j; t <= last - first; t += kSegLanes)
        s += __ldg(partial + ((long long)(first + t) * 2 + (t == 0 ? 1 : 0)) * C + c);
    part[j][threadIdx.x] = s;
    __syncthreads();
    if (j == 0 && c < C) {
      float tot = part[0][threadIdx.x];
#pragma unroll
      for (int t = 1; t < kSegLanes; ++t) tot += part[t][threadIdx.x];
      out[(long long)g * C + c] = tot;
    }
    __syncthreads();
  }
}

int segment_sum_rows(const float* data, const int* n2g, const int* graph_ptr, long long V, int G, int C, float* out,
                     cudaStream_t st) {
  if (G == 0) return 0;
  const int chunks = ceil_div(V, kSegRows);
  PoolBuffer partial{st};
  if (chunks) {
    int rc = partial.alloc((size_t)chunks * 2 * C * sizeof(float));
    if (rc) return rc;
    const bool vec = C % 4 == 0 && ((uintptr_t)data % 16) == 0 && ((uintptr_t)out % 16) == 0;
    dim3 grid((unsigned)chunks, (unsigned)ceil_div(vec ? C / 4 : C, kSegThreads));
    if (vec)
      segment_sum_chunks_kernel<true><<<grid, kSegThreads, 0, st>>>(data, n2g, graph_ptr, V, C, out, partial.f());
    else
      segment_sum_chunks_kernel<false><<<grid, kSegThreads, 0, st>>>(data, n2g, graph_ptr, V, C, out, partial.f());
    TFGNN_LAUNCH_CHECK();
  }
  dim3 grid((unsigned)(G < 132 * 8 ? G : 132 * 8), (unsigned)ceil_div(C, kSegCols));
  segment_sum_finish_kernel<<<grid, dim3(kSegCols, kSegLanes), 0, st>>>(partial.f(), graph_ptr, G, C, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// t[g,k] = sum_c grad_out[g, k*d+c] * out[g, k*d+c]  (= sum_{u in g} w[u,k] dw[u,k]: the softmax backward's per-graph term
// from the saved forward result, no walk over the graph's nodes).  One warp per (graph, head).
__global__ void readout_softmax_term_kernel(const float* __restrict__ out, const float* __restrict__ grad_out,
                                            long long GK, int d, float* __restrict__ t) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp; i < GK; i += nwarps) {
    float s = 0.f;
    for (int c = lane; c < d; c += 32) s += __ldg(grad_out + i * d + c) * __ldg(out + i * d + c);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) t[i] = s;
  }
}

// One warp per node row, heads looped, lanes over the head's d columns.  R = min(max(reprs, lower), upper);
// tf.maximum(x, lower) passes the gradient to x where x >= lower and tf.minimum(y, upper) where y <= upper (the tie goes
// to x in both), so grad_reprs is zeroed only where reprs < lower or max(reprs, lower) > upper.
__global__ void readout_bwd_kernel(const float* __restrict__ reprs, const float* __restrict__ weights,
                                   const int* __restrict__ n2g, const int* __restrict__ graph_ptr,
                                   const float* __restrict__ grad_out, const float* __restrict__ t, long long V, int GD,
                                   int K, int mode, float lo, float hi, int has_lo, int has_hi,
                                   float* __restrict__ grad_reprs, float* __restrict__ grad_scores) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int d = GD / K;
  for (long long v = warp; v < V; v += nwarps) {
    const int g = __ldg(n2g + v);
    const float* go = grad_out + (long long)g * GD;
    float unweighted = 1.f;
    if (mode == TFGNN_READOUT_AVERAGE) unweighted = 1.f / (float)max(graph_ptr[g + 1] - graph_ptr[g], 1);
    for (int k = 0; k < K; ++k) {
      const float w = weights ? __ldg(weights + v * K + k) : unweighted;
      float dw = 0.f;
      for (int c = k * d + lane; c < (k + 1) * d; c += 32) {
        const float r = __ldg(reprs + v * GD + c);
        float R = r;
        bool pass = true;
        if (has_lo) { pass = r >= lo; R = fmaxf(R, lo); }
        if (has_hi) { pass = pass && R <= hi; R = fminf(R, hi); }
        const float o = __ldg(go + c);
        dw += o * R;
        grad_reprs[v * GD + c] = pass ? w * o : 0.f;
      }
      if (!weights) continue;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dw += __shfl_xor_sync(0xffffffffu, dw, o);
      if (lane == 0)
        grad_scores[v * K + k] = mode == TFGNN_READOUT_SIGMOID ? dw * w * (1.f - w) : w * (dw - __ldg(t + (long long)g * K + k));
    }
  }
}

// ---- target-range shards: per-graph readout partials and their rank-ordered merge ------------------------------------
// The partial row of graph g (P = 2K + GD floats): K running maxima m, K sums s = sum exp(w - m) and GD weighted row sums
// S = sum exp(w - m) t (softmax); S = sum w t (sigmoid, w = 1 for none), m and s unused.  Neutral: m = -inf, s = 0, S = 0.
// Two partials combine as m = max(m1, m2), s = s1 e^(m1-m) + s2 e^(m2-m), S likewise: the online-softmax rescale of the
// RGAT hub-chunk combine.  Rows are cut into fixed kPartRows chunks (the result is a function of the rows and the cut only);
// a graph that crosses a chunk border leaves pieces in head / tail slots that the finish kernel combines in chunk order.
constexpr int kPartRows = 256, kPartThreads = 64, kPartLanes = 8, kPartCols = 32;

template <bool SOFTMAX>
__device__ __forceinline__ void part_combine(float& m, float& s, float& S, float m2, float s2, float S2) {
  if (!SOFTMAX) { S += S2; return; }
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;                 // both neutral
  const float a = expf(m - mn), b = expf(m2 - mn);
  s = s * a + s2 * b;
  S = S * a + S2 * b;
  m = mn;
}

// writes column c of a partial row: S always, m and s from the first column of each head
__device__ __forceinline__ void part_store(float* row, int c, int d, int K, float m, float s, float S) {
  row[2 * K + c] = S;
  if (c % d == 0) {
    row[c / d] = m;
    row[K + c / d] = s;
  }
}

// grid = (chunks, column tiles of kPartThreads); scratch [chunks][2][P] (head slot 0, tail slot 1)
template <bool SOFTMAX>
__global__ void __launch_bounds__(kPartThreads)
readout_partial_chunks_kernel(const float* __restrict__ w, const float* __restrict__ reprs, const int* __restrict__ n2g,
                              const int* __restrict__ graph_ptr, long long V, int GD, int K,
                              float* __restrict__ partial, float* __restrict__ scratch) {
  __shared__ int row_graph[kPartRows];
  const long long r0 = (long long)blockIdx.x * kPartRows;
  const int rows = (int)(V - r0 < kPartRows ? V - r0 : kPartRows);
  for (int j = threadIdx.x; j < rows; j += kPartThreads) row_graph[j] = __ldg(n2g + r0 + j);
  __syncthreads();
  const int c = blockIdx.y * kPartThreads + threadIdx.x;
  if (c >= GD) return;
  const int d = GD / K, k = c / d, P = 2 * K + GD;
  auto emit = [&](int g, float m, float s, float S) {
    const long long beg = graph_ptr[g], end = graph_ptr[g + 1];
    float* dst = beg < r0 ? scratch + ((long long)blockIdx.x * 2) * P
                          : (end > r0 + rows ? scratch + ((long long)blockIdx.x * 2 + 1) * P : partial + (long long)g * P);
    part_store(dst, c, d, K, m, s, S);
  };
  int cur = row_graph[0];
  float m = -INFINITY, s = 0.f, S = 0.f;
  for (int j = 0; j < rows; ++j) {
    const int g = row_graph[j];
    if (g != cur) {
      emit(cur, m, s, S);
      m = -INFINITY; s = 0.f; S = 0.f;
      cur = g;
    }
    const long long v = r0 + j;
    const float t = __ldg(reprs + v * GD + c);
    const float x = w ? __ldg(w + v * K + k) : 1.f;
    if (SOFTMAX) {
      const float mn = fmaxf(m, x);
      const float a = expf(m - mn), e = expf(x - mn);
      s = s * a + e;
      S = S * a + e * t;
      m = mn;
    } else {
      S += x * t;
    }
  }
  emit(cur, m, s, S);
}

// Graphs that cross a chunk border: the tail slot of their first chunk, then the head slots of the chunks that follow, by
// kPartLanes lanes (lane j takes pieces j, j + kPartLanes, ... in order) whose results are combined in lane order.  Graphs
// without rows get the neutral partial.  block = (kPartCols, kPartLanes); grid = (graphs, strided; column tiles)
template <bool SOFTMAX>
__global__ void __launch_bounds__(kPartCols * kPartLanes)
readout_partial_finish_kernel(const float* __restrict__ scratch, const int* __restrict__ graph_ptr, int G, int GD, int K,
                              float* __restrict__ partial) {
  __shared__ float pm[kPartLanes][kPartCols], ps[kPartLanes][kPartCols], pS[kPartLanes][kPartCols];
  const int c = blockIdx.y * kPartCols + threadIdx.x;
  const int j = threadIdx.y;
  const int d = GD / K, P = 2 * K + GD;
  for (int g = blockIdx.x; g < G; g += gridDim.x) {
    const int beg = graph_ptr[g], end = graph_ptr[g + 1];
    if (beg == end) {
      if (j == 0 && c < GD) part_store(partial + (long long)g * P, c, d, K, -INFINITY, 0.f, 0.f);
      continue;
    }
    const int first = beg / kPartRows, last = (end - 1) / kPartRows;
    if (first == last) continue;   // final since the chunk kernel
    float m = -INFINITY, s = 0.f, S = 0.f;
    if (c < GD)
      for (int t = j; t <= last - first; t += kPartLanes) {
        const float* piece = scratch + ((long long)(first + t) * 2 + (t == 0 ? 1 : 0)) * P;
        part_combine<SOFTMAX>(m, s, S, __ldg(piece + c / d), __ldg(piece + K + c / d), __ldg(piece + 2 * K + c));
      }
    pm[j][threadIdx.x] = m;
    ps[j][threadIdx.x] = s;
    pS[j][threadIdx.x] = S;
    __syncthreads();
    if (j == 0 && c < GD) {
      for (int t = 1; t < kPartLanes; ++t) part_combine<SOFTMAX>(m, s, S, pm[t][threadIdx.x], ps[t][threadIdx.x], pS[t][threadIdx.x]);
      part_store(partial + (long long)g * P, c, d, K, m, s, S);
    }
    __syncthreads();
  }
}

// One thread per (graph, column): the world's partials combined in rank order, then out = S / s (softmax) or S.
template <bool SOFTMAX>
__global__ void readout_merge_kernel(const float* __restrict__ partials, int world, int G, int GD, int K,
                                     float* __restrict__ out, float* __restrict__ gmax, float* __restrict__ gsum) {
  const int d = GD / K, P = 2 * K + GD;
  const long long total = (long long)G * GD;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long g = i / GD;
    const int c = (int)(i - g * GD), k = c / d;
    float m = -INFINITY, s = 0.f, S = 0.f;
    for (int r = 0; r < world; ++r) {
      const float* row = partials + ((long long)r * G + g) * P;
      part_combine<SOFTMAX>(m, s, S, __ldg(row + k), __ldg(row + K + k), __ldg(row + 2 * K + c));
    }
    if (SOFTMAX) {
      out[i] = s > 0.f ? S / s : 0.f;
      if (c % d == 0) {
        gmax[g * K + k] = m;
        gsum[g * K + k] = s;
      }
    } else {
      out[i] = S;
    }
  }
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_readout_partial(const float* scores, const float* node_reprs, const int32_t* node_to_graph_map,
                                          const int32_t* graph_ptr, int64_t num_rows, int32_t num_graphs, int32_t repr_dim,
                                          int32_t num_heads, int32_t mode, float* partial, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && num_rows < (1ll << 31) && num_graphs >= 0 && repr_dim > 0 && num_heads > 0 &&
                    repr_dim % num_heads == 0,
                "bad readout_partial sizes (num_heads must divide the representation size)");
  TFGNN_REQUIRE(mode >= TFGNN_READOUT_SOFTMAX && mode <= TFGNN_READOUT_NONE,
                "readout_partial: weighting mode must be softmax, sigmoid or none (average is not built for shards)");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(graph_ptr && partial, "NULL pointer");
  const bool weighted = mode != TFGNN_READOUT_NONE;
  TFGNN_REQUIRE(num_rows == 0 || (node_reprs && node_to_graph_map && (!weighted || scores)), "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const bool softmax = mode == TFGNN_READOUT_SOFTMAX;
  const int K = weighted ? num_heads : 1;
  const int chunks = ceil_div(num_rows, kPartRows);
  const int P = 2 * K + repr_dim;
  PoolBuffer scratch{st};
  if (chunks) {
    int rc = scratch.alloc((size_t)chunks * 2 * P * sizeof(float));
    if (rc) return rc;
    dim3 grid((unsigned)chunks, (unsigned)ceil_div(repr_dim, kPartThreads));
    const float* w = weighted ? scores : nullptr;
    if (softmax)
      readout_partial_chunks_kernel<true><<<grid, kPartThreads, 0, st>>>(w, node_reprs, node_to_graph_map, graph_ptr,
                                                                        num_rows, repr_dim, K, partial, scratch.f());
    else
      readout_partial_chunks_kernel<false><<<grid, kPartThreads, 0, st>>>(w, node_reprs, node_to_graph_map, graph_ptr,
                                                                         num_rows, repr_dim, K, partial, scratch.f());
    TFGNN_LAUNCH_CHECK();
  }
  dim3 grid((unsigned)(num_graphs < 132 * 8 ? num_graphs : 132 * 8), (unsigned)ceil_div(repr_dim, kPartCols));
  if (softmax)
    readout_partial_finish_kernel<true><<<grid, dim3(kPartCols, kPartLanes), 0, st>>>(scratch.f(), graph_ptr, num_graphs,
                                                                                      repr_dim, K, partial);
  else
    readout_partial_finish_kernel<false><<<grid, dim3(kPartCols, kPartLanes), 0, st>>>(scratch.f(), graph_ptr, num_graphs,
                                                                                       repr_dim, K, partial);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_readout_merge(const float* partials, int32_t world_size, int32_t num_graphs, int32_t repr_dim,
                                        int32_t num_heads, int32_t mode, float* out, float* graph_max, float* graph_sum,
                                        void* stream) {
  TFGNN_REQUIRE(world_size > 0 && num_graphs >= 0 && repr_dim > 0 && num_heads > 0 && repr_dim % num_heads == 0,
                "bad readout_merge sizes (num_heads must divide the representation size)");
  TFGNN_REQUIRE(mode >= TFGNN_READOUT_SOFTMAX && mode <= TFGNN_READOUT_NONE,
                "readout_merge: weighting mode must be softmax, sigmoid or none (average is not built for shards)");
  if (num_graphs == 0) return 0;
  const bool softmax = mode == TFGNN_READOUT_SOFTMAX;
  TFGNN_REQUIRE(partials && out && (!softmax || (graph_max && graph_sum)), "NULL pointer (softmax needs graph_max, graph_sum)");
  const int K = mode == TFGNN_READOUT_NONE ? 1 : num_heads;
  const long long total = (long long)num_graphs * repr_dim;
  cudaStream_t st = (cudaStream_t)stream;
  if (softmax)
    readout_merge_kernel<true><<<grid_for(total), 256, 0, st>>>(partials, world_size, num_graphs, repr_dim, K, out,
                                                                graph_max, graph_sum);
  else
    readout_merge_kernel<false><<<grid_for(total), 256, 0, st>>>(partials, world_size, num_graphs, repr_dim, K, out,
                                                                 nullptr, nullptr);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_segment_sum_rows(const float* data, const int32_t* node_to_graph_map, const int32_t* graph_ptr,
                                           int64_t num_rows, int32_t num_graphs, int32_t C, float* out, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && num_rows < (1ll << 31) && num_graphs >= 0 && C > 0, "bad segment_sum_rows sizes");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(graph_ptr && out, "NULL pointer");
  TFGNN_REQUIRE(num_rows == 0 || (data && node_to_graph_map), "NULL pointer");
  return segment_sum_rows(data, node_to_graph_map, graph_ptr, num_rows, num_graphs, C, out, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_readout_bwd(const float* node_reprs, const float* weights, const int32_t* node_to_graph_map,
                                      const int32_t* graph_ptr, const float* out, const float* grad_out, int64_t num_nodes,
                                      int32_t num_graphs, int32_t repr_dim, int32_t num_heads, int32_t mode, float lower,
                                      float upper, int32_t has_lower, int32_t has_upper, float* grad_reprs,
                                      float* grad_scores, void* stream) {
  TFGNN_REQUIRE(num_nodes >= 0 && num_graphs >= 0 && repr_dim > 0 && num_heads > 0 && repr_dim % num_heads == 0,
                "bad readout_bwd sizes (num_heads must divide the representation size)");
  TFGNN_REQUIRE(mode >= TFGNN_READOUT_SOFTMAX && mode <= TFGNN_READOUT_AVERAGE, "unknown readout weighting mode");
  if (num_nodes == 0) return 0;
  const bool weighted = mode == TFGNN_READOUT_SOFTMAX || mode == TFGNN_READOUT_SIGMOID;
  TFGNN_REQUIRE(node_reprs && node_to_graph_map && graph_ptr && grad_out && grad_reprs, "NULL pointer");
  TFGNN_REQUIRE(!weighted || (weights && grad_scores), "softmax / sigmoid weighting needs weights and grad_scores");
  TFGNN_REQUIRE(mode != TFGNN_READOUT_SOFTMAX || out, "softmax weighting needs the saved forward result");
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer term{st};
  if (mode == TFGNN_READOUT_SOFTMAX) {
    const long long GK = (long long)num_graphs * num_heads;
    int rc = term.alloc((size_t)GK * sizeof(float));
    if (rc) return rc;
    readout_softmax_term_kernel<<<grid_for(GK * 32), 256, 0, st>>>(out, grad_out, GK, repr_dim / num_heads, term.f());
    TFGNN_LAUNCH_CHECK();
  }
  // weights NULL: one "head" spanning the row
  readout_bwd_kernel<<<grid_for(num_nodes * 32), 256, 0, st>>>(node_reprs, weighted ? weights : nullptr, node_to_graph_map,
                                                              graph_ptr, grad_out, term.f(), num_nodes, repr_dim,
                                                              weighted ? num_heads : 1, mode, lower, upper, has_lower,
                                                              has_upper, grad_reprs, grad_scores);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

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
