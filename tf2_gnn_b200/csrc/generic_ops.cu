// The three stock ops of the reference's generic MessagePassing.call as stand-alone kernels, for
// user-defined _message_function plugins and the literal per-edge path:
//   gather_rows              = tf.nn.embedding_lookup             (message_passing.py:197-206)
//   unsorted_segment_reduce  = tf.math.unsorted_segment_{sum,mean,max,sqrt_n} (:172-174)
//   activation               = get_activation_function(name)      (:169-177)
#include "common.cuh"

namespace tfgnn {

__global__ void gather_rows_kernel(const float* __restrict__ table, long long num_rows, int D,
                                   const int* __restrict__ ids, long long ids_stride, long long n,
                                   float* __restrict__ out, int vec) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long num_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long e = warp; e < n; e += num_warps) {
    const int id = __ldg(ids + e * ids_stride);
    const bool ok = (unsigned)id < (unsigned long long)num_rows;
    const float* row = table + (long long)(ok ? id : 0) * D;
    float* o = out + e * D;
    if (vec) {
      for (int c = lane * 4; c < D; c += 128) {
        float4 v = ok ? ldg_f4(row + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(o + c) = v;
      }
    } else {
      for (int c = lane; c < D; c += 32) o[c] = ok ? __ldg(row + c) : 0.f;
    }
  }
}

__device__ __forceinline__ void atomic_max_float(float* addr, float val) {
  // total order trick: positive floats compare like ints, negative floats reversed as uints.  The branch is on
  // the SIGN BIT, not on val >= 0: -0.0f has the bit pattern 0x80000000 = INT_MIN, which atomicMax(int) would
  // never store over the -FLT_MAX identity (a segment holding only -0.0 must return -0.0, not -3.4e38).
  if (__float_as_int(val) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(val));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(val));
}

__global__ void fill_kernel(float* __restrict__ out, long long n, float v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = v;
}

__global__ void segment_scatter_kernel(const float* __restrict__ data, const int* __restrict__ ids,
                                       long long ids_stride, long long M, int H, long long num_segments,
                                       int use_max, float* __restrict__ out, int* __restrict__ counts) {
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / H;
    const int c = (int)(i - m * H);
    const int seg = __ldg(ids + m * ids_stride);
    if ((unsigned)seg >= (unsigned long long)num_segments) continue;  // TF drops out-of-range ids on GPU
    const float v = data[i];
    if (use_max) atomic_max_float(out + (long long)seg * H + c, v);
    else atomicAdd(out + (long long)seg * H + c, v);
    if (counts && c == 0) atomicAdd(counts + seg, 1);
  }
}

__global__ void segment_norm_kernel(float* __restrict__ out, const int* __restrict__ counts,
                                    long long num_segments, int H, int mode) {
  const long long total = num_segments * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const float n = (float)max(counts[i / H], 1);
    out[i] = out[i] / (mode == 1 ? n : sqrtf(n));
  }
}

__global__ void activation_kernel(const float* __restrict__ x, long long n, int act, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = apply_act(x[i], act);
}

__global__ void residual_average_kernel(const float* __restrict__ x, const float* __restrict__ last, long long n,
                                        float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = (x[i] + last[i]) / 2.0f;
}

// One warp per row; two-pass mean / variance in registers (Keras LayerNormalization: biased variance,
// y = (x - mean) * rsqrt(var + eps) * gamma + beta).
__global__ void layer_norm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, long long V, int H, float eps,
                                  float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= V) return;
  const float* xr = x + row * H;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) s += xr[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)H;
  float q = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float d = xr[c] - mean;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float inv = rsqrtf(q / (float)H + eps);
  for (int c = lane; c < H; c += 32) out[row * H + c] = (xr[c] - mean) * inv * gamma[c] + beta[c];
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_gather_rows(const float* table, int64_t num_rows, int32_t D, const int32_t* ids,
                                      int64_t ids_stride, int64_t n, float* out, void* stream) {
  TFGNN_REQUIRE(D > 0 && n >= 0 && num_rows >= 0 && ids_stride >= 1, "bad gather_rows arguments");
  if (n == 0) return 0;
  TFGNN_REQUIRE(table && ids && out, "NULL pointer");
  const int vec = (D % 4 == 0) && ((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  gather_rows_kernel<<<grid_for(n * 32), 256, 0, (cudaStream_t)stream>>>(table, num_rows, D, ids, ids_stride, n, out, vec);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_unsorted_segment_reduce(const float* data, const int32_t* segment_ids, int64_t ids_stride,
                                                  int64_t M, int32_t H, int64_t num_segments, int32_t aggregation,
                                                  float* out, void* stream) {
  TFGNN_REQUIRE(H > 0 && M >= 0 && num_segments >= 0 && ids_stride >= 1, "bad segment_reduce arguments");
  TFGNN_REQUIRE(aggregation >= TFGNN_AGG_SUM && aggregation <= TFGNN_AGG_SQRT_N, "unknown aggregation code");
  if (num_segments == 0) return 0;
  TFGNN_REQUIRE(out != nullptr, "out is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const bool use_max = aggregation == TFGNN_AGG_MAX;
  const bool need_counts = aggregation == TFGNN_AGG_MEAN || aggregation == TFGNN_AGG_SQRT_N;
  fill_kernel<<<grid_for(num_segments * H), 256, 0, st>>>(out, num_segments * H, use_max ? kLowestFloat : 0.f);
  TFGNN_LAUNCH_CHECK();
  PoolBuffer count_buf{st};
  if (need_counts) {
    int rc = count_buf.alloc((size_t)num_segments * sizeof(int));
    if (rc) return rc;
    TFGNN_CUDA(cudaMemsetAsync(count_buf.p, 0, (size_t)num_segments * sizeof(int), st));
  }
  int* counts = (int*)count_buf.p;
  if (M > 0) {
    TFGNN_REQUIRE(data && segment_ids, "NULL pointer");
    segment_scatter_kernel<<<grid_for(M * H), 256, 0, st>>>(data, segment_ids, ids_stride, M, H, num_segments,
                                                          use_max, out, counts);
    TFGNN_LAUNCH_CHECK();
  }
  if (need_counts) {
    segment_norm_kernel<<<grid_for(num_segments * H), 256, 0, st>>>(out, counts, num_segments, H,
                                                                   aggregation == TFGNN_AGG_MEAN ? 1 : 2);
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int tfgnn_b200_activation(const float* x, int64_t n, int32_t activation, float* out, void* stream) {
  TFGNN_REQUIRE(n >= 0 && activation >= TFGNN_ACT_NONE && activation <= TFGNN_ACT_SIGMOID, "bad activation arguments");
  if (n == 0) return 0;
  TFGNN_REQUIRE(x && out, "NULL pointer");
  activation_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, n, activation, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_residual_average(const float* x, const float* last, float* out, int64_t n, void* stream) {
  TFGNN_REQUIRE(n >= 0, "negative size");
  if (n == 0) return 0;
  TFGNN_REQUIRE(x && last && out, "NULL pointer");
  residual_average_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, last, n, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_layer_norm(const float* x, const float* gamma, const float* beta, int64_t V, int32_t H,
                                     float epsilon, float* out, void* stream) {
  TFGNN_REQUIRE(V >= 0 && H > 0, "bad layer_norm shape");
  if (V == 0) return 0;
  TFGNN_REQUIRE(x && gamma && beta && out, "NULL pointer");
  layer_norm_kernel<<<ceil_div(V * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, V, H, epsilon, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// ---- primitives of the differentiable generic path (layers/differentiable.py, SURVEY.md section 8f-1) -----------------
// The reference differentiates EVERY message-passing variant with tf.GradientTape through its literal op sequence
// (message_passing.py:95-218).  Variants without a fused backward (edge MLPs with two or more hidden layers, one hidden
// layer combined with max aggregation or activation before aggregation, hidden layers in GNN-FiLM's MLPs, GNN-FiLM with max
// aggregation or activation before aggregation) train through the same op sequence here: each op below is the forward or the
// backward of one TensorFlow op of that sequence.
namespace tfgnn {

// grad_in = grad_out * act'(.): `ref` is the forward OUTPUT for every activation but gelu, whose `ref` is the forward INPUT
__global__ void activation_bwd_kernel(const float* __restrict__ ref, const float* __restrict__ g, long long n, int act,
                                      float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = g[i] * (act == TFGNN_ACT_GELU ? gelu_grad_from_input(ref[i]) : act_grad_from_output(ref[i], act));
}

// out[m, :] = x[m, :] * f(s[m]),  f = s (mode 0), 1/(s + 1e-7) (mode 1: gnn_edge_mlp.py:102-106), 1/max(s,1) (mode 2:
// segment mean), 1/sqrt(max(s,1)) (mode 3: segment sqrt_n)
__global__ void row_scale_kernel(const float* __restrict__ x, const float* __restrict__ s, long long M, int H, int mode,
                                 float* __restrict__ out) {
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = s[i / H];
    const float f = mode == 0 ? v : mode == 1 ? 1.0f / (v + kSmallNumber) : mode == 2 ? 1.0f / fmaxf(v, 1.0f)
                                                                                      : 1.0f / sqrtf(fmaxf(v, 1.0f));
    out[i] = x[i] * f;
  }
}

// out = a * b + c (c NULL: a * b) over strided 2-D views: element (m, j) of each operand at ptr[m * ld + j]
__global__ void mul_add_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb,
                               const float* __restrict__ c, int ldc, long long M, int H, float* __restrict__ out, int ldo) {
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / H;
    const int j = (int)(i - m * H);
    const float v = a[m * lda + j] * b[m * ldb + j];
    out[m * ldo + j] = c ? v + c[m * ldc + j] : v;
  }
}

// backward of unsorted_segment_max: the gradient of a segment's maximum goes to the messages that attain it
// (ties share the whole gradient each, as tf.math.unsorted_segment_max's gradient does through its equality mask / count:
//  the count normalisation is applied too)
__global__ void segment_max_bwd_kernel(const float* __restrict__ data, const int* __restrict__ ids, long long ids_stride,
                                       const float* __restrict__ seg_out, const float* __restrict__ seg_grad,
                                       const float* __restrict__ tie_count, long long M, int H,
                                       long long num_segments, float* __restrict__ out) {
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / H;
    const int c = (int)(i - m * H);
    const int seg = ids[m * ids_stride];
    float g = 0.f;
    if ((unsigned)seg < (unsigned long long)num_segments && data[i] == seg_out[(long long)seg * H + c])
      g = seg_grad[(long long)seg * H + c] / fmaxf(tie_count[(long long)seg * H + c], 1.0f);
    out[i] = g;
  }
}
__global__ void segment_max_ties_kernel(const float* __restrict__ data, const int* __restrict__ ids, long long ids_stride,
                                        const float* __restrict__ seg_out, long long M, int H, long long num_segments,
                                        float* __restrict__ tie_count) {
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / H;
    const int c = (int)(i - m * H);
    const int seg = ids[m * ids_stride];
    if ((unsigned)seg < (unsigned long long)num_segments && data[i] == seg_out[(long long)seg * H + c])
      atomicAdd(tie_count + (long long)seg * H + c, 1.0f);
  }
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_activation_bwd(const float* ref, const float* grad_out, int64_t n, int32_t activation,
                                         float* grad_in, void* stream) {
  TFGNN_REQUIRE(n >= 0 && activation >= TFGNN_ACT_NONE && activation <= TFGNN_ACT_SIGMOID, "bad activation_bwd arguments");
  if (n == 0) return 0;
  TFGNN_REQUIRE(ref && grad_out && grad_in, "NULL pointer");
  activation_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(ref, grad_out, n, activation, grad_in);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_row_scale(const float* x, const float* s, int64_t M, int32_t H, int32_t mode, float* out,
                                    void* stream) {
  TFGNN_REQUIRE(M >= 0 && H > 0 && mode >= 0 && mode <= 3, "bad row_scale arguments");
  if (M == 0) return 0;
  TFGNN_REQUIRE(x && s && out, "NULL pointer");
  row_scale_kernel<<<grid_for(M * H), 256, 0, (cudaStream_t)stream>>>(x, s, M, H, mode, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_mul_add(const float* a, int32_t lda, const float* b, int32_t ldb, const float* c, int32_t ldc,
                                  int64_t M, int32_t H, float* out, int32_t ldo, void* stream) {
  TFGNN_REQUIRE(M >= 0 && H > 0, "bad mul_add arguments");
  if (M == 0) return 0;
  TFGNN_REQUIRE(a && b && out, "NULL pointer");
  mul_add_kernel<<<grid_for(M * H), 256, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, c, ldc, M, H, out, ldo);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_segment_max_bwd(const float* data, const int32_t* segment_ids, int64_t ids_stride,
                                          const float* segment_out, const float* segment_grad, int64_t M, int32_t H,
                                          int64_t num_segments, float* grad_data, void* stream) {
  TFGNN_REQUIRE(M >= 0 && H > 0 && num_segments >= 0 && ids_stride >= 1, "bad segment_max_bwd arguments");
  if (M == 0) return 0;
  TFGNN_REQUIRE(data && segment_ids && segment_out && segment_grad && grad_data, "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer ties{st};
  int rc = ties.alloc((size_t)num_segments * H * sizeof(float));
  if (rc) return rc;
  TFGNN_CUDA(cudaMemsetAsync(ties.p, 0, (size_t)num_segments * H * sizeof(float), st));
  segment_max_ties_kernel<<<grid_for(M * H), 256, 0, st>>>(data, segment_ids, ids_stride, segment_out, M, H, num_segments,
                                                          ties.f());
  TFGNN_LAUNCH_CHECK();
  segment_max_bwd_kernel<<<grid_for(M * H), 256, 0, st>>>(data, segment_ids, ids_stride, segment_out, segment_grad,
                                                         ties.f(), M, H, num_segments, grad_data);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// ---- attention / softmax pieces of the differentiable generic path (rgat.py:133-160, nodes_to_graph_representation.py:176-227)
namespace tfgnn {

// out = exp(s - m)                      (z == nullptr)
// out = exp((s - m) - log(z))           (dpu_utils unsorted_segment_log_softmax, then tf.exp: rgat.py:147-151)
__global__ void softmax_apply_kernel(const float* __restrict__ s, const float* __restrict__ m, const float* __restrict__ z,
                                     long long n, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float r = s[i] - m[i];
    out[i] = z ? expf(r - logf(z[i])) : expf(r);
  }
}

// out[e, k*d + i] = w[e, k] * x[e, k*d + i]     (tf.expand_dims(attention, -1) * messages, rgat.py:152-155)
__global__ void head_scale_kernel(const float* __restrict__ x, const float* __restrict__ w, long long M, int K, int d,
                                  float* __restrict__ out) {
  const int H = K * d;
  const long long total = M * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i / H;
    const int k = (int)(i - e * H) / d;
    out[i] = w[e * K + k] * x[i];
  }
}

// out[e, k] = sum_i a[e, k*d + i] * b[e, k*d + i]   (gradient of head_scale with respect to the weights)
__global__ void head_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, long long M, int K, int d,
                                float* __restrict__ out) {
  const long long total = M * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i / K;
    const int k = (int)(i - e * K);
    const float* pa = a + e * (long long)K * d + (long long)k * d;
    const float* pb = b + e * (long long)K * d + (long long)k * d;
    float s = 0.f;
    for (int j = 0; j < d; ++j) s = fmaf(pa[j], pb[j], s);
    out[i] = s;
  }
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_softmax_apply(const float* scores, const float* seg_max_per_elem, const float* seg_sum_per_elem,
                                        int64_t n, float* out, void* stream) {
  TFGNN_REQUIRE(n >= 0, "negative size");
  if (n == 0) return 0;
  TFGNN_REQUIRE(scores && seg_max_per_elem && out, "NULL pointer");
  softmax_apply_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(scores, seg_max_per_elem, seg_sum_per_elem, n, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_head_scale(const float* x, const float* w, int64_t M, int32_t num_heads, int32_t head_dim,
                                     float* out, void* stream) {
  TFGNN_REQUIRE(M >= 0 && num_heads > 0 && head_dim > 0, "bad head_scale arguments");
  if (M == 0) return 0;
  TFGNN_REQUIRE(x && w && out, "NULL pointer");
  head_scale_kernel<<<grid_for(M * num_heads * head_dim), 256, 0, (cudaStream_t)stream>>>(x, w, M, num_heads, head_dim, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_head_dot(const float* a, const float* b, int64_t M, int32_t num_heads, int32_t head_dim, float* out,
                                   void* stream) {
  TFGNN_REQUIRE(M >= 0 && num_heads > 0 && head_dim > 0, "bad head_dot arguments");
  if (M == 0) return 0;
  TFGNN_REQUIRE(a && b && out, "NULL pointer");
  head_dot_kernel<<<grid_for(M * num_heads), 256, 0, (cudaStream_t)stream>>>(a, b, M, num_heads, head_dim, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}
