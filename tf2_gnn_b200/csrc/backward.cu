// Backward pass of the RGCN-style layer (SURVEY.md §8f-1): the reference differentiates through the layer
// with tf.GradientTape (tf2_gnn/models/graph_task_model.py:338-365); here the gradients of
//     out = act( rn(v) * sum_l A_l W_l ),   A_l[v] = s_{v,l} * sum_{(u,v) in A_l} h_u,   s = 1/(c_{v,l}+eps) or 1
// are computed with the same building blocks as the forward pass:
//   dZ      = dOut * act'(out) * rn(v)                        (elementwise, from the saved OUTPUT)
//   dW_l    = A_l^T dZ                                        (A recomputed by the CSR reduce; TN GEMM, reduction
//                                                              over the V nodes in fixed chunks -> deterministic)
//   dA      = dZ [W_0;..;W_{L-1}]^T, then dA_l[v] *= s_{v,l}   (3xTF32 wgmma GEMM + row/type scale)
//   dh[u]   = sum_l sum_{(u,v) in A_l} dA_l[v]                (CSR reduce over the SOURCE-keyed CSR: no atomics)
// Supported: 0 hidden layers, source or source+target state input, sum / mean / sqrt_n aggregation, activation after the
// aggregation, every activation of the reference's table (gelu through a recomputed pre-activation).  Max aggregation and
// activation before the aggregation take the transform-then-aggregate backward (transform_aggregate_bwd, below).
// On a target-range shard (DESIGN.md §6) everything but the dh reduce covers the owned rows only; the dh reduce runs over the
// shard's TFGNN_PREPARE_TRANSPOSE_OWNED CSR (all global sources, local target ids), so each shard writes its contribution
// to the full grad_h table and the contributions of all shards sum to the unsharded gradient.
#include <initializer_list>

#include "layers.cuh"

namespace tfgnn {

// ties (max aggregation): the tie count n of every (v, c); dz is then divided by it, as tf.math.unsorted_segment_max's
// gradient divides by its count (segment_max_bwd_kernel), and is 0 where n = 0 (a target without edges carries no gradient).
__global__ void act_grad_kernel(const float* __restrict__ g, const float* __restrict__ out, long long V, int H,
                                int act, const int* __restrict__ row_ptr, int L, int row_norm,
                                float* __restrict__ dz, const float* __restrict__ ties = nullptr) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    float s = 1.f;
    if (row_norm) {
      int cnt = 0;
      for (int l = 0; l < L; ++l) cnt += row_ptr[(long long)l * V + v + 1] - row_ptr[(long long)l * V + v];
      const float n = (float)max(cnt, 1);
      s = 1.f / (row_norm == 1 ? n : sqrtf(n));
    }
    // for gelu `out` holds the recomputed pre-activation
    const float d = g[i] * (act == TFGNN_ACT_GELU ? gelu_grad_from_input(out[i]) : act_grad_from_output(out[i], act)) * s;
    dz[i] = ties ? (ties[i] > 0.f ? d / ties[i] : 0.f) : d;
  }
}

// dA[v, l*D + c] *= 1/(c_{v,l}+eps)   (first L*D columns of rows with leading dimension ld)
__global__ void scale_by_type_kernel(float* __restrict__ dA, int ld, long long V, int L, int D,
                                     const int* __restrict__ row_ptr) {
  const long long total = V * L * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / ((long long)L * D);
    const int col = (int)(i - v * (long long)L * D);
    const int l = col / D;
    const long long seg = (long long)l * V + v;
    dA[v * ld + col] *= 1.0f / ((float)(row_ptr[seg + 1] - row_ptr[seg]) + kSmallNumber);
  }
}

// use_target_state_as_input (gnn_edge_mlp.py:93-98): the target half of the node-level operand is
// T[v, l*D + c] = coeff(v,l) * h_v[c], coeff = c/(c+eps) or c; its gradient flows straight back to h_v:
// grad_h[v, c] += sum_l coeff(v,l) * dT[v, l*D + c]
__global__ void target_term_bwd_kernel(const float* __restrict__ dT, int ld, const int* __restrict__ row_ptr, long long V,
                                       int L, int D, int normalize, float* __restrict__ grad_h) {
  const long long total = V * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / D;
    const int c = (int)(i - v * D);
    float s = 0.f;
    for (int l = 0; l < L; ++l) {
      const long long seg = (long long)l * V + v;
      const float cnt = (float)(row_ptr[seg + 1] - row_ptr[seg]);
      const float coeff = normalize ? cnt * (1.0f / (cnt + kSmallNumber)) : cnt;
      s += coeff * dT[v * ld + (long long)l * D + c];
    }
    grad_h[i] += s;
  }
}

// WcatT[hh, col0 + l*D + d] = W_l[row0 + d, hh]   (operand of dA = dZ Wcat^T; ld_out = columns of WcatT)
__global__ void pack_transposed_kernel(PtrTable W, int L, int D, int H, float* __restrict__ out, int ld_out = 0,
                                       int col0 = 0, int row0 = 0) {
  const long long total = (long long)L * D * H;
  if (ld_out == 0) ld_out = L * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % ((long long)L * D));
    const int hh = (int)(i / ((long long)L * D));
    const int l = col / D, d = col - l * D;
    out[(long long)hh * ld_out + col0 + col] = reinterpret_cast<const float*>(W.p[l])[(long long)(row0 + d) * H + hh];
  }
}

// TN GEMM with the reduction over the (huge) node dimension: Cpart[chunk][k][n] = sum_{m in chunk} A[m,k] B[m,n].
// 128x128 output tile, 256 threads, 8x8 per thread; both operands are read row-wise (row m contiguous), so no
// transposition is needed in shared memory.  fp32 FFMA (deterministic; a tensor-core version is future work).
constexpr int kTnTile = 128, kTnMB = 16, kTnChunk = 8192;

__global__ void __launch_bounds__(256, 2)
gemm_tn_partial_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, long long M,
                       int Kd, int N, float* __restrict__ Cpart) {
  // 16-byte row loads need 4-float leading dimensions and aligned bases (rgcn_bwd guarantees them; the Dense backward
  // of e.g. a 50-feature input layer does not)
  const bool vecA = (lda & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0;
  const bool vecB = (ldb & 3) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0;
  __shared__ __align__(16) float As[2][kTnMB][kTnTile];
  __shared__ __align__(16) float Bs[2][kTnMB][kTnTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int k0 = blockIdx.x * kTnTile, n0 = blockIdx.y * kTnTile;
  const long long m_begin = (long long)blockIdx.z * kTnChunk;
  const long long m_end = m_begin + kTnChunk < M ? m_begin + kTnChunk : M;
  const int lr = t >> 5, lc = (t & 31) * 4;     // load coordinates: rows lr, lr+8 ; 4 consecutive columns
  float4 ra[2], rb[2];
  auto load = [&](long long m0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long m = m0 + lr + 8 * i;
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
      if (m < m_end) {
        const float* pa = A + m * lda + k0 + lc;
        const float* pb = B + m * ldb + n0 + lc;
        if (vecA && k0 + lc + 3 < Kd) va = __ldg(reinterpret_cast<const float4*>(pa));
        else {
          if (k0 + lc < Kd) va.x = pa[0];
          if (k0 + lc + 1 < Kd) va.y = pa[1];
          if (k0 + lc + 2 < Kd) va.z = pa[2];
          if (k0 + lc + 3 < Kd) va.w = pa[3];
        }
        if (vecB && n0 + lc + 3 < N) vb = __ldg(reinterpret_cast<const float4*>(pb));
        else {
          if (n0 + lc < N) vb.x = pb[0];
          if (n0 + lc + 1 < N) vb.y = pb[1];
          if (n0 + lc + 2 < N) vb.z = pb[2];
          if (n0 + lc + 3 < N) vb.w = pb[3];
        }
      }
      ra[i] = va;
      rb[i] = vb;
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      *reinterpret_cast<float4*>(&As[buf][lr + 8 * i][lc]) = ra[i];
      *reinterpret_cast<float4*>(&Bs[buf][lr + 8 * i][lc]) = rb[i];
    }
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  load(m_begin);
  store(0);
  __syncthreads();
  int buf = 0;
  for (long long m0 = m_begin; m0 < m_end; m0 += kTnMB, buf ^= 1) {
    if (m0 + kTnMB < m_end) load(m0 + kTnMB);
#pragma unroll
    for (int mm = 0; mm < kTnMB; ++mm) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][mm][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][mm][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][mm][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][mm][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (m0 + kTnMB < m_end) {
      store(buf ^ 1);
      __syncthreads();
    }
  }
  float* cp = Cpart + (long long)blockIdx.z * Kd * N;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = k0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (k >= Kd) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n < N) cp[(long long)k * N + n] = acc[i][j];
    }
  }
}

// dW_l[d, :] = sum over chunks of Cpart[chunk][l*D + d, :]   (fixed order: deterministic)
// Cpart rows [k0, k0 + L*D) of K_total rows per chunk (K_total = 0: L*D) go to rows [row0, row0 + D) of dW_l.
__global__ void reduce_partials_kernel(const float* __restrict__ Cpart, int chunks, int L, int D, int N,
                                       PtrTable dW, int K_total = 0, int k0 = 0, int row0 = 0) {
  const long long total = (long long)L * D * N;
  if (K_total == 0) K_total = L * D;
  const long long chunk_stride = (long long)K_total * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += Cpart[(long long)c * chunk_stride + (long long)k0 * N + i];
    const int row = (int)(i / N), n = (int)(i - (long long)row * N);
    const int l = row / D, d = row - l * D;
    reinterpret_cast<float*>(const_cast<void*>(dW.p[l]))[(long long)(row0 + d) * N + n] = s;
  }
}

// ---- GGNN: Keras GRUCell (reset_after=True) backward, ggnn.py:84-87 -------------------------------------------------
// forward: z = sig(gx_z+gh_z), r = sig(gx_r+gh_r), hh = tanh(gx_h + r*gh_h), h' = z*h + (1-z)*hh.
// dgx = dL/dgx, dgh = dL/dgh, dh_direct = dL/dh' * z (the path of h through the convex combination).  dgx / dgh may be
// gx / gh (GGNN's backward works in place): each thread reads its six pre-activations before it writes.  gx_index
// (optional) picks row gx_index[v] of gx as gru_gate_kernel does; dgx is per node either way.
__global__ void gru_gate_bwd_kernel(const float* gx, const int* __restrict__ gx_index, const float* gh,
                                    const float* __restrict__ h, int ldh, const float* __restrict__ grad_out, long long V,
                                    int H, float* dgx, float* dgh, float* __restrict__ dh_direct) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    const int c = (int)(i - v * H);
    const float* x = gx + (gx_index ? (long long)__ldg(gx_index + v) : v) * 3 * H;
    const float* y = gh + v * 3 * H;
    const float ghh = y[2 * H + c];
    const float hv = h[v * ldh + c];
    const float z = 1.0f / (1.0f + expf(-(x[c] + y[c])));
    const float r = 1.0f / (1.0f + expf(-(x[H + c] + y[H + c])));
    const float hh = tanhf(x[2 * H + c] + r * ghh);
    const float g = grad_out[i];
    const float da = g * (1.0f - z) * (1.0f - hh * hh);   // d/d(pre-tanh)
    const float daz = g * (hv - hh) * z * (1.0f - z);
    const float dar = da * ghh * r * (1.0f - r);
    float* ox = dgx + v * 3 * H;
    float* oy = dgh + v * 3 * H;
    ox[c] = daz;          oy[c] = daz;
    ox[H + c] = dar;      oy[H + c] = dar;
    ox[2 * H + c] = da;   oy[2 * H + c] = da * r;
    dh_direct[i] = g * z;
  }
}

// column sums over the node dimension in fixed 8192-row chunks (deterministic): partial[chunk][n]
__global__ void colsum_partial_kernel(const float* __restrict__ X, long long V, int N, float* __restrict__ partial) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const long long m0 = (long long)blockIdx.y * kTnChunk;
  const long long m1 = m0 + kTnChunk < V ? m0 + kTnChunk : V;
  float s = 0.f;
  for (long long m = m0; m < m1; ++m) s += X[m * N + n];
  partial[(long long)blockIdx.y * N + n] = s;
}
__global__ void colsum_reduce_kernel(const float* __restrict__ partial, int chunks, int N, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += partial[(long long)c * N + n];
  out[n] = s;
}

// grad_h = grad_h (message path) + a + b
__global__ void add3_kernel(float* __restrict__ acc, const float* __restrict__ a, const float* __restrict__ b, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc[i] = acc[i] + a[i] + b[i];
}

// (b, bt) of a backward call: the unsharded pair (bt = TFGNN_PREPARE_TRANSPOSE of the same graph) or a target-range shard
// and its TFGNN_PREPARE_TRANSPOSE_OWNED batch over the same range.
static int check_backward_pair(const tfgnn_batch* b, const tfgnn_batch* bt) {
  const bool sharded = b->tgt_off != 0 || b->V_src != b->V;
  TFGNN_REQUIRE(!b->owned_transpose, "the first batch of a backward call must be the forward (target-keyed) batch");
  if (sharded)
    TFGNN_REQUIRE(bt->owned_transpose && bt->own_begin == b->tgt_off && bt->own_count == b->V && bt->V == b->V_src &&
                      bt->L == b->L,
                  "a target-range shard needs its TFGNN_PREPARE_TRANSPOSE_OWNED batch over the same range");
  else
    TFGNN_REQUIRE(bt->V == b->V && bt->L == b->L && bt->V_src == b->V && (!bt->owned_transpose || bt->own_count == b->V),
                  "forward and transposed batches must describe the same graph");
  return 0;
}

static PtrTable one_table(const void* p) {
  PtrTable t{};
  t.p[0] = p;
  return t;
}

static int tn_chunks(long long M) { return (int)((M + kTnChunk - 1) / kTnChunk); }
// floats of the partial buffer of weight_grad over M rows
static size_t tn_partial_floats(long long M, int Kd, int N) { return (size_t)tn_chunks(M) * Kd * N; }

// Weight gradient X^T Y for X [M, Kd], Y [M, N]: partial sums over fixed kTnChunk-row chunks, then summed in chunk order, so
// the result is bitwise reproducible.  `part` holds tn_partial_floats(M, Kd, N).  The rows of X^T Y come in blocks of D:
// block j goes to rows [row0 + (j / L) D, row0 + (j / L + 1) D) of dW_{j % L}.
static int weight_grad(const float* X, int ldx, const float* Y, int ldy, long long M, int Kd, int N, float* part,
                       PtrTable dW, int L, int D, int row0, cudaStream_t st) {
  const int chunks = tn_chunks(M);
  gemm_tn_partial_kernel<<<dim3(ceil_div(Kd, kTnTile), ceil_div(N, kTnTile), chunks), 256, 0, st>>>(X, ldx, Y, ldy, M, Kd,
                                                                                                      N, part);
  TFGNN_LAUNCH_CHECK();
  for (int k0 = 0; k0 < Kd; k0 += L * D) {
    reduce_partials_kernel<<<grid_for((long long)L * D * N), 256, 0, st>>>(part, chunks, L, D, N, dW, Kd, k0,
                                                                            row0 + k0 / L);
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

// The transposes of a table of L weights W_l (H columns each), as packed for gemm_transposed: rows
// [row0 + p D, row0 + (p + 1) D) of every W_l for p < parts, transposed.  Side by side: WT [H, parts L D] with block (p, l) at
// column (p L + l) D.  Stacked (parts = 1): WT [L H, D] with block l at row l H.
struct TransposedWeights {
  PtrTable W;
  int L, D, H;
  int parts = 1, row0 = 0;
  bool stacked = false;
};

// C [M, N] = X WT (epilogue `epi`, node GEMM) after packing WT (pack_transposed_kernel): X [M, H] multiplies every type's
// block side by side; stacked, X [M, L H] holds one block per type and the product sums over the types.
static int gemm_transposed(const float* X, int ldx, const TransposedWeights& w, float* WT, float* C, int ldc, long long M,
                           int N, const GemmEpilogue& epi, cudaStream_t st) {
  if (w.stacked) {
    for (int l = 0; l < w.L; ++l) {
      pack_transposed_kernel<<<grid_for((long long)w.D * w.H), 256, 0, st>>>(one_table(w.W.p[l]), 1, w.D, w.H,
                                                                             WT + (size_t)l * w.H * w.D, w.D, 0, w.row0);
      TFGNN_LAUNCH_CHECK();
    }
    return node_gemm(X, ldx, WT, w.D, C, ldc, M, N, w.L * w.H, epi, TFGNN_PATH_AUTO, st);
  }
  const int LD = w.L * w.D;
  for (int p = 0; p < w.parts; ++p) {
    pack_transposed_kernel<<<grid_for((long long)LD * w.H), 256, 0, st>>>(w.W, w.L, w.D, w.H, WT, w.parts * LD, p * LD,
                                                                          w.row0 + p * w.D);
    TFGNN_LAUNCH_CHECK();
  }
  return node_gemm(X, ldx, WT, w.parts * LD, C, ldc, M, N, w.H, epi, TFGNN_PATH_AUTO, st);
}

// n gradient buffers p[0], p[step], p[2 step], .. of `floats` floats each
struct GradBuffers {
  float* const* p;
  int n;
  size_t floats;
  int step = 1;
};

// The contribution of a backward call without owned rows (an empty shard) or without edge types: every weight gradient and
// grad_h (when given, grad_h_floats floats) are cleared.
static int zero_contribution(std::initializer_list<GradBuffers> weights, float* grad_h, size_t grad_h_floats,
                             cudaStream_t st) {
  for (const GradBuffers& g : weights)
    for (int i = 0; i < g.n; ++i) {
      float* p = g.p[(size_t)i * g.step];
      TFGNN_REQUIRE(p, "a weight-gradient pointer is NULL");
      TFGNN_CUDA(cudaMemsetAsync(p, 0, g.floats * sizeof(float), st));
    }
  if (grad_h && grad_h_floats) TFGNN_CUDA(cudaMemsetAsync(grad_h, 0, grad_h_floats * sizeof(float), st));
  return 0;
}

static int enter_both(tfgnn_batch* b, tfgnn_batch* bt, cudaStream_t st) {
  const int rc = batch_enter(b, st);
  return rc ? rc : batch_enter(bt, st);
}

// The start of a fused layer backward with owned rows and edge types: enters both batches and forms
// dZ = dOut * act'(out) * rn(v) [V, H] in the caller's buffer dz.  For gelu, act' needs the pre-activation: `preact(z)`
// recomputes it (the layer's forward without activation) into a pool buffer that is freed once dZ is formed.
template <class Preact>
static int begin_backward(tfgnn_batch* b, tfgnn_batch* bt, const float* out, const float* grad_out, int H, int activation,
                          int aggregation, cudaStream_t st, PoolBuffer& dz, Preact preact) {
  const long long V = b->V;
  int rc = enter_both(b, bt, st);
  if (rc) return rc;
  PoolBuffer z{st};
  if (activation == TFGNN_ACT_GELU) {
    rc = z.alloc((size_t)V * H * sizeof(float));
    if (!rc) rc = preact(z.f());
    if (rc) return rc;
    out = z.f();
  }
  rc = dz.alloc((size_t)V * H * sizeof(float));
  if (rc) return rc;
  act_grad_kernel<<<grid_for(V * H), 256, 0, st>>>(grad_out, out, V, H, activation, b->row_ptr, b->L,
                                                   agg_row_norm(aggregation), dz.f());
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// grad_h[u] = sum over the edges LEAVING u of every type l of dA_l[v] (at dA + v ldx + l D): the merged reduce over bt's
// source-keyed CSR.  On a shard that is its owned transpose: Vs segments per type (every global source; rows without an
// owned edge get zeros), values = local target ids = rows of dA.
static int reduce_over_sources(const tfgnn_batch* bt, const float* dA, int ldx, int D, long long Vs, float* grad_h,
                               cudaStream_t st) {
  EdgeReduceParams p;
  p.X = dA; p.ldx = ldx; p.x_type_stride = D;
  p.row_ptr = bt->row_ptr; p.src = bt->src_sorted;
  p.out = grad_h; p.ldo = D;
  p.V = (int)Vs; p.L = bt->L; p.C = D;
  return launch_edge_reduce(p, /*merged=*/true, st);
}

// column sums of X [V, N] in fixed-order chunks -> out [N]   (bias / gamma / beta gradients).  `part` holds
// tn_chunks(V) * N floats; without it the call takes a pool buffer.
static int column_sums(const float* X, long long V, int N, float* out, float* part, cudaStream_t st) {
  const int chunks = tn_chunks(V);
  PoolBuffer own{st};
  if (!part) {
    const int rc = own.alloc((size_t)chunks * N * sizeof(float));
    if (rc) return rc;
    part = own.f();
  }
  colsum_partial_kernel<<<dim3(ceil_div(N, 128), chunks), 128, 0, st>>>(X, V, N, part);
  TFGNN_LAUNCH_CHECK();
  colsum_reduce_kernel<<<ceil_div(N, 128), 128, 0, st>>>(part, chunks, N, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// Backward of the transform-then-aggregate form (no hidden layer, max aggregation and / or activation before aggregation;
// DESIGN.md §6).  Per edge e = (u -> v) of type l: x_e = (P_l[u] + T_l[v]) s, y_e = act_edge(x_e), z[v] = agg_e y_e,
// out = act_final(rn(v) z), with P = h [W_0|..], T = h_tgt [W^t_0|..] (target-state input, else 0):
//   1. P, T recomputed by the forward's node GEMMs (transform_aggregate_tables); for max, z and the tie count n in one pass
//      of the forward's edge reduce
//   2. dZ = dOut * act_final'(z) / n  (max)   or   dOut * rn(v)  (sum / mean / sqrt_n: act_final is the identity)
//   3. w_e = dZ[v] * [y_e == z[v]] (max) * act_edge'(x_e) (activation before) * s;  dP_l[u] = sum_{e leaving u} w_e over
//      the source-keyed CSR, dT_l[v] = sum_{e into v} w_e over the forward's CSR (edge_grad_kernel, one template)
//   4. dW_l = h^T dP_l,  dW^t_l = h_tgt^T dT_l   (TN, fixed 8192-row chunks)
//   5. grad_h = dP [W_0^T; ..] (+ dT [W^t_0^T; ..] on the owned rows)
// Every temporary is [V or Vs, L*H] at most.  On a shard, dP and grad_h cover every source (bt is the owned transpose), dT and
// the target term the owned rows.
static int transform_aggregate_bwd(tfgnn_batch* b, tfgnn_batch* bt, const float* h, int D, const PtrTable& wt,
                                   float* const* grad_W, int H, uint32_t flags, int aggregation, int activation,
                                   const float* out, const float* grad_out, float* grad_h, cudaStream_t st) {
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L, LH = L * H;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;
  const bool use_max = aggregation == TFGNN_AGG_MAX;
  int rc = enter_both(b, bt, st);
  if (rc) return rc;
  // 1. P, T and (max) z, n
  EdgeReduceParams f;
  PoolBuffer P{st}, T{st};
  rc = transform_aggregate_tables(b, h, D, wt, H, flags, aggregation, activation, TFGNN_PATH_AUTO, P, T, &f, st);
  if (rc) return rc;
  const int final_act = f.final_act;
  PoolBuffer zn{st}, dz{st}, dP{st}, dT{st};
  if (use_max) {
    rc = zn.alloc((size_t)2 * V * H * sizeof(float));   // z, then n
    if (rc) return rc;
    EdgeReduceParams p = f;
    p.out = zn.f(); p.ldo = H; p.final_act = TFGNN_ACT_NONE; p.ties = zn.f() + (size_t)V * H;
    rc = launch_edge_reduce(p, /*merged=*/true, st);
    if (rc) return rc;
  }
  const float* z = use_max ? zn.f() : nullptr;
  rc = dz.alloc((size_t)V * H * sizeof(float));
  if (rc) return rc;
  // 2. dZ (act_final' from the saved output, or for gelu from z)
  act_grad_kernel<<<grid_for(V * H), 256, 0, st>>>(grad_out, final_act == TFGNN_ACT_GELU ? z : out, V, H, final_act,
                                                   b->row_ptr, L, f.row_norm, dz.f(),
                                                   use_max ? z + (size_t)V * H : nullptr);
  TFGNN_LAUNCH_CHECK();
  // 3. dP over the source-keyed CSR, dT over the forward's
  rc = dP.alloc((size_t)Vs * LH * sizeof(float));
  if (rc) return rc;
  rc = launch_edge_grad(f, z, dz.f(), bt->row_ptr, bt->src_sorted, (int)Vs, dP.f(), st);
  if (rc) return rc;
  if (use_target) {
    rc = dT.alloc((size_t)V * LH * sizeof(float));
    if (rc) return rc;
    rc = launch_edge_grad(f, z, dz.f(), nullptr, nullptr, 0, dT.f(), st);
    if (rc) return rc;
  }
  // 4. dW_l over all Vs rows, dW^t_l (rows [D, 2D) of W_l) over the owned rows
  const float* h_tgt = h + (size_t)lo * D;
  {
    PoolBuffer part{st};
    rc = part.alloc(tn_partial_floats(Vs, D, H) * sizeof(float));   // Vs >= V
    if (rc) return rc;
    for (int l = 0; l < L; ++l) {
      const PtrTable gw = one_table(grad_W[l]);
      rc = weight_grad(h, D, dP.f() + (size_t)l * H, LH, Vs, D, H, part.f(), gw, 1, D, 0, st);
      if (rc) return rc;
      if (use_target) {
        rc = weight_grad(h_tgt, D, dT.f() + (size_t)l * H, LH, V, D, H, part.f(), gw, 1, D, D, st);
        if (rc) return rc;
      }
    }
  }
  if (!grad_h) return 0;
  // 5. grad_h = dP [W_0^T; ..] (K = L*H), then the owned rows += dT [W^t_0^T; ..]
  PoolBuffer WT{st};
  rc = WT.alloc((size_t)LH * D * sizeof(float));
  if (!rc) rc = gemm_transposed(dP.f(), LH, {wt, L, D, H, 1, 0, /*stacked=*/true}, WT.f(), grad_h, D, Vs, D,
                                GemmEpilogue{}, st);
  if (rc || !use_target) return rc;
  GemmEpilogue acc;
  acc.accumulate = 1;
  return gemm_transposed(dT.f(), LH, {wt, L, D, H, 1, D, /*stacked=*/true}, WT.f(), grad_h + (size_t)lo * D, D, V, D,
                         acc, st);
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_rgcn_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D,
                                   const float* const* W, int32_t H, uint32_t flags, int32_t aggregation,
                                   int32_t activation, const float* out, const float* grad_out, float* grad_h,
                                   float* const* grad_W, void* stream) {
  TFGNN_REQUIRE(b != nullptr && bt != nullptr, "batch / transposed batch is NULL");
  TFGNN_REQUIRE(D > 0 && H > 0, "D and H must be positive");
  TFGNN_REQUIRE(valid_act(activation) && valid_agg(aggregation), "unknown activation / aggregation code");
  // V = owned target rows (of out / grad_out), Vs = rows of h and grad_h, lo = global id of local target 0
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L;
  if (int rc = check_backward_pair(b, bt)) return rc;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;   // W_l is then [2D, H]: rows [0,D) source, [D,2D) target
  const bool transform_aggregate = aggregation == TFGNN_AGG_MAX || (flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION);
  if (D % 4 != 0 || H % 4 != 0) return unsupported("rgcn_bwd needs D and H to be multiples of 4");
  if (transform_aggregate && H > 512)
    return unsupported("rgcn_bwd: max aggregation / activation before aggregation above hidden_dim 512 is not built");
  TFGNN_REQUIRE(L == 0 || (W && grad_W), "weight / weight-gradient table is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0 || L == 0)   // no owned rows (an empty shard) or no edge types: zero contribution
    return zero_contribution({{grad_W, L, (size_t)(use_target ? 2 * D : D) * H}}, grad_h, (size_t)Vs * D, st);
  TFGNN_REQUIRE(h && out && grad_out, "NULL pointer");
  const float* h_tgt = h + (size_t)lo * D;   // rows of the owned targets (target-state input)
  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const int LD = L * D;
  const int K = use_target ? 2 * LD : LD;
  PtrTable wt{}, gwt{};
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(W[l] && grad_W[l], "a weight pointer is NULL");
    wt.p[l] = W[l];
    gwt.p[l] = grad_W[l];
  }
  if (transform_aggregate)
    return transform_aggregate_bwd(b, bt, h, D, wt, grad_W, H, flags, aggregation, activation, out, grad_out, grad_h, st);
  // 1. dZ = dOut * act'(out) * rn(v)
  PoolBuffer dz{st};
  int rc = begin_backward(b, bt, out, grad_out, H, activation, aggregation, st, dz, [&](float* z) {
    return edge_mlp_core(b, h, D, W, 0, H, flags, aggregation, TFGNN_ACT_NONE, TFGNN_PATH_AUTO, z, H, st);
  });
  if (rc) return rc;
  PoolBuffer A{st};   // A (forward operand), then dA
  rc = A.alloc((size_t)V * K * sizeof(float));
  if (rc) return rc;

  // 2. A_l (recomputed, normalised) and dW = A^T dZ
  {
    EdgeReduceParams p;
    p.X = h; p.ldx = D; p.x_type_stride = 0;
    p.row_ptr = b->row_ptr; p.src = b->src_sorted;
    p.out = A.f(); p.ldo = K; p.out_type_stride = D;
    p.V = (int)V; p.L = L; p.C = D; p.normalize = normalize;
    rc = launch_edge_reduce(p, /*merged=*/false, st);
    if (rc) return rc;
  }
  if (use_target) {
    rc = launch_target_term(h_tgt, D, b->row_ptr, (int)V, L, D, normalize, A.f(), K, LD, st);
    if (rc) return rc;
  }
  {
    PoolBuffer part{st};
    rc = part.alloc(tn_partial_floats(V, K, H) * sizeof(float));
    if (!rc) rc = weight_grad(A.f(), K, dz.f(), H, V, K, H, part.f(), gwt, L, D, 0, st);
    if (rc || !grad_h) return rc;
  }
  // 3. dA = dZ Wcat^T (overwrites A), scaled per (v,l)
  {
    PoolBuffer WT{st};
    rc = WT.alloc((size_t)K * H * sizeof(float));
    if (!rc) rc = gemm_transposed(dz.f(), H, {wt, L, D, H, use_target ? 2 : 1}, WT.f(), A.f(), K, V, K, GemmEpilogue{}, st);
    if (rc) return rc;
  }
  if (normalize) {
    scale_by_type_kernel<<<grid_for(V * LD), 256, 0, st>>>(A.f(), K, V, L, D, b->row_ptr);
    TFGNN_LAUNCH_CHECK();
  }
  // 4. dh[u] = sum over the edges LEAVING u
  rc = reduce_over_sources(bt, A.f(), K, D, Vs, grad_h, st);
  if (rc) return rc;
  if (use_target) {   // 5. the target half: grad_h[lo + v] += sum_l coeff(v,l) * dT_l[v]
    target_term_bwd_kernel<<<grid_for(V * D), 256, 0, st>>>(A.f() + LD, K, b->row_ptr, V, L, D, normalize,
                                                            grad_h + (size_t)lo * D);
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

namespace tfgnn {

// Backward of the GRU update out = GRUCell(agg, h) over V rows (gru_update), from the given agg:
//   1. gx = agg K + b0, gh = h U + b1 (tensor-core GEMMs);  2. gate backward in place -> dgx, dgh, dh_direct;
//   3. db = column sums;  4. dK = agg^T dgx, dU = h^T dgh (TN GEMM, fixed-order partials);
//   5. dagg = dgx K^T, dh_rec = dgh U^T (tensor-core GEMMs).
// dh_rec == nullptr: the recurrent term is added onto dh_direct instead.  Every temporary is freed on return.
static int gru_update_bwd(const float* agg, const float* h, int ldh, const float* gru_kernel,
                          const float* gru_recurrent_kernel, const float* gru_bias, const float* grad_out, long long V, int H,
                          float* dagg, float* dh_direct, float* dh_rec, float* grad_gru_kernel,
                          float* grad_gru_recurrent_kernel, float* grad_gru_bias, cudaStream_t st) {
  const int N3 = 3 * H;
  PoolBuffer gx{st}, gh{st}, wT{st}, part{st};
  int rc = gx.alloc((size_t)V * N3 * sizeof(float));
  if (!rc) rc = gh.alloc((size_t)V * N3 * sizeof(float));
  if (!rc) rc = wT.alloc((size_t)N3 * H * sizeof(float));
  if (!rc) rc = part.alloc((tn_partial_floats(V, H, N3) + (size_t)tn_chunks(V) * N3) * sizeof(float));
  if (rc) return rc;
  // 1. forward quantities gx, gh
  GemmEpilogue e0, e1;
  e0.bias = gru_bias;
  e1.bias = gru_bias + N3;
  rc = node_gemm(agg, H, gru_kernel, N3, gx.f(), N3, V, N3, H, e0, TFGNN_PATH_AUTO, st);
  if (rc) return rc;
  rc = node_gemm(h, ldh, gru_recurrent_kernel, N3, gh.f(), N3, V, N3, H, e1, TFGNN_PATH_AUTO, st);
  if (rc) return rc;
  // 2. gates, in place
  gru_gate_bwd_kernel<<<grid_for(V * H), 256, 0, st>>>(gx.f(), nullptr, gh.f(), h, ldh, grad_out, V, H, gx.f(), gh.f(),
                                                       dh_direct);
  TFGNN_LAUNCH_CHECK();
  // 3. bias gradients: rows 0 / 1 of gru_bias belong to gx / gh
  float* cpart = part.f() + tn_partial_floats(V, H, N3);
  rc = column_sums(gx.f(), V, N3, grad_gru_bias, cpart, st);
  if (rc) return rc;
  rc = column_sums(gh.f(), V, N3, grad_gru_bias + N3, cpart, st);
  if (rc) return rc;
  // 4. dK = agg^T dgx, dU = h^T dgh
  rc = weight_grad(agg, H, gx.f(), N3, V, H, N3, part.f(), one_table(grad_gru_kernel), 1, H, 0, st);
  if (rc) return rc;
  rc = weight_grad(h, ldh, gh.f(), N3, V, H, N3, part.f(), one_table(grad_gru_recurrent_kernel), 1, H, 0, st);
  if (rc) return rc;
  // 5. dagg = dgx K^T, dh_rec = dgh U^T
  rc = gemm_transposed(gx.f(), N3, {one_table(gru_kernel), 1, H, N3}, wT.f(), dagg, H, V, H, GemmEpilogue{}, st);
  if (rc) return rc;
  GemmEpilogue rec;
  rec.accumulate = dh_rec == nullptr;
  return gemm_transposed(gh.f(), N3, {one_table(gru_recurrent_kernel), 1, H, N3}, wT.f(), dh_rec ? dh_rec : dh_direct, H, V,
                         H, rec, st);
}

}  // namespace tfgnn

// GGNN backward (SURVEY.md section 8f-1): gradient of tfgnn_b200_ggnn_fwd w.r.t. the node states, the per-type message
// weights and the GRU parameters.  Everything is recomputed from h (nothing but h is saved by the forward pass):
//   agg = sum_l s A_l W_l (forward kernel), then the GRU update's backward (gru_update_bwd) -> dagg, dh_direct, dh_rec and
//   the GRU gradients;  messages: tfgnn_b200_rgcn_bwd with dagg.
extern "C" int tfgnn_b200_ggnn_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D,
                                   const float* const* W, int32_t H, uint32_t flags, int32_t aggregation,
                                   const float* gru_kernel, const float* gru_recurrent_kernel, const float* gru_bias,
                                   const float* grad_out, float* grad_h, float* const* grad_W, float* grad_gru_kernel,
                                   float* grad_gru_recurrent_kernel, float* grad_gru_bias, void* stream) {
  TFGNN_REQUIRE(b != nullptr && bt != nullptr, "batch / transposed batch is NULL");
  TFGNN_REQUIRE(D == H, "GGNN needs node embedding dimension == hidden_dim (ggnn.py:30)");
  TFGNN_REQUIRE(valid_agg(aggregation), "unknown aggregation code");
  // V = owned target rows, Vs = rows of h and grad_h; the GRU state of local row v is h[lo + v]
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L;
  if (int rc = check_backward_pair(b, bt)) return rc;
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;   // W_l is then [2D, H], as for tfgnn_b200_rgcn_bwd
  if (H % 4 != 0) return unsupported("ggnn_bwd needs hidden_dim to be a multiple of 4");
  if (aggregation == TFGNN_AGG_MAX && H > 512)
    return unsupported("ggnn_bwd: max aggregation above hidden_dim 512 is not built");
  TFGNN_REQUIRE(grad_h, "NULL pointer");
  TFGNN_REQUIRE(grad_gru_kernel && grad_gru_recurrent_kernel && grad_gru_bias, "GRU gradient pointer is NULL");
  TFGNN_REQUIRE(L == 0 || grad_W, "weight-gradient table is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const int N3 = 3 * H;
  if (V == 0)   // no owned rows (an empty shard): zero contribution
    return zero_contribution({{&grad_gru_kernel, 1, (size_t)H * N3},
                              {&grad_gru_recurrent_kernel, 1, (size_t)H * N3},
                              {&grad_gru_bias, 1, (size_t)2 * N3},
                              {grad_W, L, (size_t)(use_target ? 2 * D : D) * H}},
                             grad_h, (size_t)Vs * D, st);
  TFGNN_REQUIRE(h && grad_out, "NULL pointer");
  TFGNN_REQUIRE(gru_kernel && gru_recurrent_kernel && gru_bias, "GRU weight pointer is NULL");
  int rc = enter_both(b, bt, st);
  if (rc) return rc;
  PoolBuffer dagg{st}, dhd{st}, tmp{st};
  rc = dagg.alloc((size_t)V * H * sizeof(float));
  if (!rc) rc = dhd.alloc((size_t)V * H * sizeof(float));
  if (!rc) rc = tmp.alloc((size_t)V * H * sizeof(float));
  if (rc) return rc;
  {
    // agg and the GRU's own temporaries are freed before the message backward below
    PoolBuffer agg{st};
    rc = agg.alloc((size_t)V * H * sizeof(float));
    if (rc) return rc;
    // agg: no message activation (ggnn.py:68-83)
    rc = edge_mlp_core(b, h, D, W, 0, H, flags & ~TFGNN_FLAG_ACT_BEFORE_AGGREGATION, aggregation, TFGNN_ACT_NONE,
                       TFGNN_PATH_AUTO, agg.f(), H, st);
    if (!rc) rc = gru_update_bwd(agg.f(), h + (size_t)lo * D, D, gru_kernel, gru_recurrent_kernel, gru_bias, grad_out, V, H,
                                 dagg.f(), dhd.f(), tmp.f(), grad_gru_kernel, grad_gru_recurrent_kernel, grad_gru_bias, st);
    if (rc) return rc;
  }
  // 6. messages: dagg -> grad_h (through the edges) and grad_W
  rc = tfgnn_b200_rgcn_bwd(b, bt, h, D, W, H, flags & ~TFGNN_FLAG_ACT_BEFORE_AGGREGATION, aggregation, TFGNN_ACT_NONE,
                           dagg.f(), dagg.f(), grad_h, grad_W, stream);
  if (rc) return rc;
  // 7. grad_h[lo + v] += dh_direct + dh_rec
  add3_kernel<<<grid_for(V * H), 256, 0, st>>>(grad_h + (size_t)lo * D, dhd.f(), tmp.f(), V * H);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_gru_update_bwd(const float* agg, const float* h, int64_t num_rows, int32_t H,
                                         const float* gru_kernel, const float* gru_recurrent_kernel, const float* gru_bias,
                                         const float* grad_out, float* grad_agg, float* grad_h, float* grad_gru_kernel,
                                         float* grad_gru_recurrent_kernel, float* grad_gru_bias, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && H > 0, "bad gru_update_bwd sizes");
  if (H % 4 != 0) return unsupported("gru_update_bwd needs hidden_dim to be a multiple of 4");
  TFGNN_REQUIRE(grad_gru_kernel && grad_gru_recurrent_kernel && grad_gru_bias, "GRU gradient pointer is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const int N3 = 3 * H;
  if (num_rows == 0)
    return zero_contribution({{&grad_gru_kernel, 1, (size_t)H * N3},
                              {&grad_gru_recurrent_kernel, 1, (size_t)H * N3},
                              {&grad_gru_bias, 1, (size_t)2 * N3}},
                             nullptr, 0, st);
  TFGNN_REQUIRE(agg && h && grad_out && grad_agg && grad_h, "NULL pointer");
  TFGNN_REQUIRE(gru_kernel && gru_recurrent_kernel && gru_bias, "GRU weight pointer is NULL");
  return gru_update_bwd(agg, h, H, gru_kernel, gru_recurrent_kernel, gru_bias, grad_out, num_rows, H, grad_agg, grad_h,
                        nullptr, grad_gru_kernel, grad_gru_recurrent_kernel, grad_gru_bias, st);
}

extern "C" int tfgnn_b200_gru_gate_bwd(const float* gx, const float* gh, const float* h, const float* grad_out,
                                       int64_t num_rows, int32_t H, float* grad_gx, float* grad_gh, float* grad_h_direct,
                                       void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && H > 0, "bad gru_gate_bwd sizes");
  if (num_rows == 0) return 0;
  TFGNN_REQUIRE(gx && gh && h && grad_out && grad_gx && grad_gh && grad_h_direct, "NULL pointer");
  gru_gate_bwd_kernel<<<grid_for(num_rows * H), 256, 0, (cudaStream_t)stream>>>(gx, nullptr, gh, h, H, grad_out, num_rows,
                                                                               H, grad_gx, grad_gh, grad_h_direct);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// The GRU exchange's backward: gx = graph_repr K + b0 has one row per GRAPH, so grad_gx is the per-node gate gradient summed
// over each graph's rows (tfgnn_b200_segment_sum_rows): the input-side GEMMs of the cell stay G-row GEMMs in the backward too.
extern "C" int tfgnn_b200_gru_gate_bwd_indexed(const float* gx, const int32_t* node_to_graph_map, const int32_t* graph_ptr,
                                               const float* gh, const float* h, const float* grad_out, int64_t num_rows,
                                               int32_t num_graphs, int32_t H, float* grad_gx, float* grad_gh,
                                               float* grad_h_direct, void* stream) {
  TFGNN_REQUIRE(num_rows >= 0 && num_rows < (1ll << 31) && num_graphs >= 0 && H > 0, "bad gru_gate_bwd_indexed sizes");
  if (num_graphs == 0) return 0;
  TFGNN_REQUIRE(graph_ptr && grad_gx, "NULL pointer");
  TFGNN_REQUIRE(num_rows == 0 || (gx && node_to_graph_map && gh && h && grad_out && grad_gh && grad_h_direct),
                "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer dgx{st};
  if (num_rows) {
    int rc = dgx.alloc((size_t)num_rows * 3 * H * sizeof(float));
    if (rc) return rc;
    gru_gate_bwd_kernel<<<grid_for(num_rows * H), 256, 0, st>>>(gx, node_to_graph_map, gh, h, H, grad_out, num_rows, H,
                                                               dgx.f(), grad_gh, grad_h_direct);
    TFGNN_LAUNCH_CHECK();
  }
  return tfgnn_b200_segment_sum_rows(dgx.f(), node_to_graph_map, graph_ptr, num_rows, num_graphs, 3 * H, grad_gx, stream);
}

// =====================================================================================================================
// GNN-FiLM backward in the aggregate-then-transform form of tfgnn_b200_film_fwd (variants.cu, DESIGN.md §3).  Per target v
// and type l, with c = c_{v,l}, s = 1/(c+eps) or 1, A_l = s sum_e h_u, T_l = c s h_v, [gamma_l | beta_l] = h_v F_l:
//   Q_l = A_l W^s_l (+ T_l W^t_l),   Z = sum_l gamma_l * Q_l + c beta_l,   out = act(rn(v) Z)
// and with dZ = dOut * act' * rn(v):
//   dQ_l = dZ * gamma_l        (GEMM h_v Fgamma_l, epilogue mul = dZ)
//   dgamma_l = dZ * Q_l        (GEMM [A_l | T_l] W_l, epilogue mul = dZ),   dbeta_l = c dZ
//   dW_l = [A_l | T_l]^T dQ_l,   dF_l = h_v^T [dgamma_l | dbeta_l]          (TN, fixed 8192-row chunks)
//   dA_l = s dQ_l W^s_l^T       -> grad_h[u] through the source-keyed CSR (all types merged, no atomics)
//   grad_h[v] += [dgamma_l | dbeta_l] F_l^T (+ c s dQ_l W^t_l^T)            (owned rows)
// Every per-type temporary is [V, D], [V, H] or [V, 2H]; only dA holds all types ([V, L*D]).
// =====================================================================================================================
namespace tfgnn {

// dGB[v, H + c] = c_{v,l} * dZ[v, c]: the beta half of [dgamma_l | dbeta_l] (row_ptr_l = the CSR offsets of type l), next to
// the gamma half so that one TN pass gives dF_l
__global__ void film_beta_grad_kernel(const float* __restrict__ dz, const int* __restrict__ row_ptr_l, long long V, int H,
                                      float* __restrict__ dgb) {
  const long long total = V * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / H;
    const int c = (int)(i - v * H);
    dgb[v * 2 * H + H + c] = (float)(row_ptr_l[v + 1] - row_ptr_l[v]) * dz[i];
  }
}

// acc += a
__global__ void add_kernel(float* __restrict__ acc, const float* __restrict__ a, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc[i] += a[i];
}

}  // namespace tfgnn

namespace tfgnn {

// The shared body of tfgnn_b200_film_bwd and tfgnn_b200_film_in_bwd.  The FiLM MLPs' last layers read fin [V, L*S] (owned
// rows): type l reads columns [l*fstride, l*fstride + S).  fstride 0 (film_bwd): fin is ignored and h's owned rows [V, D]
// are read instead, S = D, and the
// FiLM term [dgamma_l | dbeta_l] F_l^T lands in grad_h with the target-state term.  Else it goes to grad_fin [V, L*S] (may be
// NULL) and grad_h gets the message side and the target-state term only.  `name` prefixes the unsupported-case messages.
static int film_bwd_core(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int D, const float* const* mlp_weights,
                         const float* fin, int fstride, int S, const float* const* film_weights, int H,
                         uint32_t flags, int aggregation, int activation, const float* out, const float* grad_out,
                         float* grad_h, float* grad_fin, float* const* grad_W, float* const* grad_film, const char* name,
                         cudaStream_t st) {
  // the configuration is judged from the scalar arguments alone, before any batch is read
  const std::string who(name);
  const std::string dims = fstride ? "D, H and S" : "D and H";
  TFGNN_REQUIRE(D > 0 && H > 0 && S > 0, who + ": " + dims + " must be positive");
  TFGNN_REQUIRE(valid_act(activation) && valid_agg(aggregation), who + ": unknown activation / aggregation code");
  if (flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION)
    return unsupported(who + ": activation-before-aggregation is not built yet");
  if (aggregation == TFGNN_AGG_MAX) return unsupported(who + ": max aggregation is not built yet");
  if (D % 4 != 0 || H % 4 != 0 || S % 4 != 0)
    return unsupported(who + " needs " + dims + " to be multiples of 4");
  TFGNN_REQUIRE(b != nullptr && bt != nullptr, who + ": batch / transposed batch is NULL");
  // V = owned target rows (of out / grad_out), Vs = rows of h and grad_h, lo = global id of local target 0
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L;
  if (int rc = check_backward_pair(b, bt)) return rc;
  TFGNN_REQUIRE((long long)L * S < (1ll << 31), who + ": L * S overflows");
  const int ldf = fstride ? L * S : D;   // columns of fin and grad_fin
  TFGNN_REQUIRE(L == 0 || (mlp_weights && film_weights && grad_W && grad_film), "weight / weight-gradient table is NULL");
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;   // W_l is then [2D, H]: rows [0,D) source, [D,2D) target
  const int KT = use_target ? 2 * D : D;                          // columns of [A_l | T_l], rows of W_l
  for (int l = 0; l < L; ++l)
    TFGNN_REQUIRE(mlp_weights[l] && film_weights[l] && grad_W[l] && grad_film[l], "a weight pointer is NULL");
  if (V == 0 || L == 0)   // no owned rows (an empty shard) or no edge types: zero contribution
    return zero_contribution({{grad_W, L, (size_t)KT * H}, {grad_film, L, (size_t)S * 2 * H}}, grad_h, (size_t)Vs * D, st);
  const float* h_tgt = h ? h + (size_t)lo * D : nullptr;   // rows of the owned targets (target-state input)
  if (!fstride) fin = h_tgt;
  TFGNN_REQUIRE(h && out && grad_out && fin, who + ": NULL pointer");
  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const bool film_to_h = fstride == 0;       // the FiLM input is h itself: its gradient term goes to grad_h
  if (film_to_h) grad_fin = nullptr;
  const bool target_side = grad_h && (film_to_h || use_target);   // grad_h gets owned-row terms (dHt)
  const int LD = L * D, SD = S > D ? S : D;
  // 1. dZ = dOut * act'(out) * rn(v)
  PoolBuffer dz{st};
  int rc = begin_backward(b, bt, out, grad_out, H, activation, aggregation, st, dz, [&](float* z) {
    return film_fwd_core(b, h, D, mlp_weights, 0, fin, fstride, S, film_weights, H, flags, aggregation,
                         TFGNN_ACT_NONE, TFGNN_PATH_AUTO, z, st);
  });
  if (rc) return rc;
  PoolBuffer AT{st}, dQ{st}, dGB{st}, part{st};
  rc = AT.alloc((size_t)V * KT * sizeof(float));                                       // [A_l | T_l], later dT_l
  if (!rc) rc = dQ.alloc((size_t)V * H * sizeof(float));
  if (!rc) rc = dGB.alloc((size_t)V * 2 * H * sizeof(float));                          // [dgamma_l | dbeta_l]
  if (!rc) rc = part.alloc(tn_partial_floats(V, SD, 2 * H) * sizeof(float));   // KT * H <= D * 2H
  if (rc) return rc;
  PoolBuffer dA{st}, dHt{st}, WT{st}, FT{st};
  if (grad_h) {
    rc = dA.alloc((size_t)V * LD * sizeof(float));
    if (!rc && target_side) rc = dHt.alloc((size_t)V * D * sizeof(float));   // target-side terms of grad_h, summed over types
    if (!rc) rc = WT.alloc((size_t)H * KT * sizeof(float));
    if (rc) return rc;
    if (!film_to_h && use_target) TFGNN_CUDA(cudaMemsetAsync(dHt.f(), 0, (size_t)V * D * sizeof(float), st));
  }
  if ((grad_h && film_to_h) || grad_fin) {
    rc = FT.alloc((size_t)2 * H * S * sizeof(float));
    if (rc) return rc;
  }

  GemmEpilogue none, by_dz;
  by_dz.mul = dz.f();
  by_dz.ldm = H;
  for (int l = 0; l < L; ++l) {
    const int* rp = b->row_ptr + (size_t)l * V;   // the V segments of type l
    const float* Wl = mlp_weights[l];
    const float* Fl = film_weights[l];
    const float* zl = fin + (size_t)l * fstride;   // type l's FiLM input
    // 2. [A_l | T_l] (recomputed)
    {
      EdgeReduceParams p;
      p.X = h; p.ldx = D; p.x_type_stride = 0;
      p.row_ptr = rp; p.src = b->src_sorted;
      p.out = AT.f(); p.ldo = KT; p.out_type_stride = 0;
      p.V = (int)V; p.L = 1; p.C = D; p.normalize = normalize;
      rc = launch_edge_reduce(p, /*merged=*/false, st);
      if (rc) return rc;
      if (use_target) {
        rc = launch_target_term(h_tgt, D, rp, (int)V, 1, D, normalize, AT.f(), KT, D, st);
        if (rc) return rc;
      }
    }
    // 3. dQ_l = dZ * (z_l Fgamma_l);  dgamma_l = dZ * ([A_l | T_l] W_l);  dbeta_l = c dZ
    rc = node_gemm(zl, ldf, Fl, 2 * H, dQ.f(), H, V, H, S, by_dz, TFGNN_PATH_AUTO, st);
    if (rc) return rc;
    rc = node_gemm(AT.f(), KT, Wl, H, dGB.f(), 2 * H, V, H, KT, by_dz, TFGNN_PATH_AUTO, st);
    if (rc) return rc;
    film_beta_grad_kernel<<<grid_for(V * H), 256, 0, st>>>(dz.f(), rp, V, H, dGB.f());
    TFGNN_LAUNCH_CHECK();
    // 4. dW_l = [A_l | T_l]^T dQ_l,  dF_l = z_l^T [dgamma_l | dbeta_l]
    rc = weight_grad(AT.f(), KT, dQ.f(), H, V, KT, H, part.f(), one_table(grad_W[l]), 1, KT, 0, st);
    if (rc) return rc;
    rc = weight_grad(zl, ldf, dGB.f(), 2 * H, V, S, 2 * H, part.f(), one_table(grad_film[l]), 1, S, 0, st);
    if (rc) return rc;
    if (grad_fin) {   // dz_l = [dgamma_l | dbeta_l] F_l^T into type l's columns of grad_fin
      rc = gemm_transposed(dGB.f(), 2 * H, {one_table(Fl), 1, S, 2 * H}, FT.f(), grad_fin + (size_t)l * fstride, ldf, V,
                           S, none, st);
      if (rc) return rc;
    }
    if (!grad_h) continue;
    // 5. dA_l = dQ_l W^s_l^T into columns [l*D, (l+1)*D) of dA (scaled by s after the loop)
    rc = gemm_transposed(dQ.f(), H, {one_table(Wl), 1, KT, H}, WT.f(), dA.f() + (size_t)l * D, LD, V, D, none, st);
    if (rc) return rc;
    // 6. target side: dHt (+)= [dgamma_l | dbeta_l] F_l^T (film_to_h) (+ coeff(v,l) dQ_l W^t_l^T)
    if (film_to_h) {
      GemmEpilogue sum_types;
      sum_types.accumulate = l > 0;
      rc = gemm_transposed(dGB.f(), 2 * H, {one_table(Fl), 1, D, 2 * H}, FT.f(), dHt.f(), D, V, D, sum_types, st);
      if (rc) return rc;
    }
    if (use_target) {   // dT_l overwrites [A_l | T_l] (read for the last time by the dW_l pass above); W^t_l^T is packed
      rc = node_gemm(dQ.f(), H, WT.f() + D, KT, AT.f(), KT, V, D, H, none, TFGNN_PATH_AUTO, st);
      if (rc) return rc;
      target_term_bwd_kernel<<<grid_for(V * D), 256, 0, st>>>(AT.f(), KT, rp, V, 1, D, normalize, dHt.f());
      TFGNN_LAUNCH_CHECK();
    }
  }
  if (!grad_h) return 0;
  if (normalize) {
    scale_by_type_kernel<<<grid_for(V * LD), 256, 0, st>>>(dA.f(), LD, V, L, D, b->row_ptr);
    TFGNN_LAUNCH_CHECK();
  }
  // 7. grad_h[u] = sum over the edges LEAVING u
  rc = reduce_over_sources(bt, dA.f(), LD, D, Vs, grad_h, st);
  if (rc) return rc;
  if (!target_side) return 0;
  // 8. grad_h[lo + v] += target-side terms
  add_kernel<<<grid_for(V * D), 256, 0, st>>>(grad_h + (size_t)lo * D, dHt.f(), V * D);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_film_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D,
                                   const float* const* mlp_weights, const float* const* film_weights, int32_t H,
                                   uint32_t flags, int32_t aggregation, int32_t activation, const float* out,
                                   const float* grad_out, float* grad_h, float* const* grad_W, float* const* grad_film,
                                   void* stream) {
  return film_bwd_core(b, bt, h, D, mlp_weights, nullptr, 0, D, film_weights, H, flags, aggregation, activation, out,
                       grad_out, grad_h, nullptr, grad_W, grad_film, "film_bwd", (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_film_in_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D,
                                      const float* const* mlp_weights, const float* film_in, int32_t S,
                                      const float* const* film_weights, int32_t H, uint32_t flags, int32_t aggregation,
                                      int32_t activation, const float* out, const float* grad_out, float* grad_h,
                                      float* grad_film_in, float* const* grad_W, float* const* grad_film, void* stream) {
  return film_bwd_core(b, bt, h, D, mlp_weights, film_in, S, S, film_weights, H, flags, aggregation, activation,
                       out, grad_out, grad_h, grad_film_in, grad_W, grad_film, "film_in_bwd", (cudaStream_t)stream);
}

// =====================================================================================================================
// Edge MLP with one hidden layer (GNN_Edge_MLP defaults, RGIN defaults) in the hoisted form of tfgnn_b200_edge_mlp_fwd
// (api.cu, DESIGN.md §3).  Per edge e = (u -> v) of type l, with Xs = h [U^s_0 | ..], Xt = h_v [U^t_0 | ..] (target-state
// input only, else 0), P_e = Xs_l[u] + Xt_l[v], m_e = [P_e > 0] (TF ReluGrad: the derivative at 0 is 0):
//   A_l[v] = s_{v,l} sum_e relu(P_e),   out = act(rn(v) [A_0 | ..] [W2_0; ..])
// and with dZ = dOut * act' * rn(v):
//   dW2_l = A_l^T dZ                                   (A recomputed; TN, fixed 8192-row chunks)
//   dA = dZ [W2_0; ..]^T, dA_l[v] *= s_{v,l}           (one [V, L*H] GEMM)
//   dXs_l[u] = sum_{e leaving u, type l} dA_l[v] m_e   (source-keyed CSR, one warp per (type, source), no atomics)
//   dXt_l[v] = dA_l[v] * cnt_l[v],  cnt_l[v, c] = sum_{e into v} m_e[c]   (counted in the recompute pass)
//   dU^s_l = h^T dXs_l,  dU^t_l = h_v^T dXt_l          (TN)
//   grad_h = dXs [U^s_0^T; ..] (+ dXt [U^t_0^T; ..] on the owned rows)
// Every temporary is [V or Vs, L*H] at most; nothing has a per-edge dimension.
// =====================================================================================================================
namespace tfgnn {

// A_l[v] and cnt_l[v] for target-state input: one warp per (type, target) segment.  The edge order per lane, the sum and
// the end-of-segment scale are those of the forward's hidden_relu edge reduce, so A has the forward's bits.  All tables
// have L*H columns.
template <int NV>
__global__ void __launch_bounds__(256) hidden_relu_count_kernel(const float* __restrict__ Xs, const float* __restrict__ Xt,
                                                                const int* __restrict__ row_ptr, const int* __restrict__ src,
                                                                int V, int L, int H, int normalize, float* __restrict__ A,
                                                                float* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const long long ld = (long long)L * H;
  const int C4 = H >> 2;
  const long long items = (long long)L * V;
  for (long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < items;
       item += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int l = (int)(item / V), v = (int)(item - (long long)l * V);
    const int beg = __ldg(row_ptr + item), end = __ldg(row_ptr + item + 1);
    const long long col = (long long)l * H;
    float4 t[NV], acc[NV], n[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c4 = lane + 32 * j;
      t[j] = (c4 < C4 && end > beg) ? ldg_f4(Xt + v * ld + col + 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[j] = n[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int base = beg; base < end; base += 32) {
      const int m = min(32, end - base);
      const int my_src = lane < m ? __ldg(src + base + lane) : 0;
#pragma unroll 1   // unrolled, the three float4 accumulator sets spill at NV = 3, 4
      for (int e = 0; e < m; ++e) {
        const float* row = Xs + (long long)__shfl_sync(0xffffffffu, my_src, e) * ld + col;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const int c4 = lane + 32 * j;
          if (c4 >= C4) continue;
          const float4 r = ldg_f4(row + 4 * c4);
          const float4 x = make_float4(r.x + t[j].x, r.y + t[j].y, r.z + t[j].z, r.w + t[j].w);
          acc[j] = make_float4(acc[j].x + fmaxf(x.x, 0.f), acc[j].y + fmaxf(x.y, 0.f), acc[j].z + fmaxf(x.z, 0.f),
                               acc[j].w + fmaxf(x.w, 0.f));
          n[j] = make_float4(n[j].x + (x.x > 0.f ? 1.f : 0.f), n[j].y + (x.y > 0.f ? 1.f : 0.f),
                             n[j].z + (x.z > 0.f ? 1.f : 0.f), n[j].w + (x.w > 0.f ? 1.f : 0.f));
        }
      }
    }
    const float s = normalize ? 1.0f / ((float)(end - beg) + kSmallNumber) : 1.0f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c4 = lane + 32 * j;
      if (c4 >= C4) continue;
      float4 a = acc[j];
      if (normalize) a = make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
      *reinterpret_cast<float4*>(A + v * ld + col + 4 * c4) = make_float4(0.f + a.x, 0.f + a.y, 0.f + a.z, 0.f + a.w);
      *reinterpret_cast<float4*>(cnt + v * ld + col + 4 * c4) = n[j];
    }
  }
}

// dXs_l[u] = sum over the edges (u -> v) of type l of dA_l[v] * m_e, over the source-keyed CSR (row_ptr_t: segment
// (l, u) = l*Vs + u; tgt: local target ids), in canonical order, one warp per segment.  Xs_l[u] stays in registers.
// Without target-state input (TGT = false) m_e = [Xs_l[u] > 0] is the same for every edge of the segment: applied once.
template <int NV, bool TGT>
__global__ void __launch_bounds__(256) hidden_relu_src_bwd_kernel(const float* __restrict__ Xs, const float* __restrict__ Xt,
                                                                  const float* __restrict__ dA,
                                                                  const int* __restrict__ row_ptr_t,
                                                                  const int* __restrict__ tgt, int Vs, int L, int H,
                                                                  float* __restrict__ dXs) {
  const int lane = threadIdx.x & 31;
  const long long ld = (long long)L * H;
  const int C4 = H >> 2;
  const long long items = (long long)L * Vs;
  for (long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < items;
       item += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int l = (int)(item / Vs), u = (int)(item - (long long)l * Vs);
    const int beg = __ldg(row_ptr_t + item), end = __ldg(row_ptr_t + item + 1);
    const long long col = (long long)l * H;
    float4 xs[NV], acc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c4 = lane + 32 * j;
      xs[j] = (c4 < C4 && end > beg) ? ldg_f4(Xs + u * ld + col + 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int base = beg; base < end; base += 32) {
      const int m = min(32, end - base);
      const int my_tgt = lane < m ? __ldg(tgt + base + lane) : 0;
#pragma unroll 4
      for (int e = 0; e < m; ++e) {
        const long long off = (long long)__shfl_sync(0xffffffffu, my_tgt, e) * ld + col;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const int c4 = lane + 32 * j;
          if (c4 >= C4) continue;
          const float4 g = ldg_f4(dA + off + 4 * c4);
          if (TGT) {
            const float4 t = ldg_f4(Xt + off + 4 * c4);
            acc[j].x += (xs[j].x + t.x > 0.f) ? g.x : 0.f;
            acc[j].y += (xs[j].y + t.y > 0.f) ? g.y : 0.f;
            acc[j].z += (xs[j].z + t.z > 0.f) ? g.z : 0.f;
            acc[j].w += (xs[j].w + t.w > 0.f) ? g.w : 0.f;
          } else {
            acc[j] = make_float4(acc[j].x + g.x, acc[j].y + g.y, acc[j].z + g.z, acc[j].w + g.w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c4 = lane + 32 * j;
      if (c4 >= C4) continue;
      float4 a = acc[j];
      if (!TGT)
        a = make_float4(xs[j].x > 0.f ? a.x : 0.f, xs[j].y > 0.f ? a.y : 0.f, xs[j].z > 0.f ? a.z : 0.f,
                        xs[j].w > 0.f ? a.w : 0.f);
      *reinterpret_cast<float4*>(dXs + u * ld + col + 4 * c4) = a;
    }
  }
}

// x *= y
__global__ void mul_inplace_kernel(float* __restrict__ x, const float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] *= y[i];
}

static int warp_grid(long long items) {
  const long long g = (items * 32 + 255) / 256;
  return g < 1 ? 1 : (g > 132 * 64 ? 132 * 64 : (int)g);
}

static int launch_hidden_relu_count(const float* Xs, const float* Xt, const int* row_ptr, const int* src, int V, int L,
                                    int H, int normalize, float* A, float* cnt, cudaStream_t st) {
  const int g = warp_grid((long long)L * V);
  switch ((H + 127) / 128) {
    case 1: hidden_relu_count_kernel<1><<<g, 256, 0, st>>>(Xs, Xt, row_ptr, src, V, L, H, normalize, A, cnt); break;
    case 2: hidden_relu_count_kernel<2><<<g, 256, 0, st>>>(Xs, Xt, row_ptr, src, V, L, H, normalize, A, cnt); break;
    case 3: hidden_relu_count_kernel<3><<<g, 256, 0, st>>>(Xs, Xt, row_ptr, src, V, L, H, normalize, A, cnt); break;
    case 4: hidden_relu_count_kernel<4><<<g, 256, 0, st>>>(Xs, Xt, row_ptr, src, V, L, H, normalize, A, cnt); break;
    default: return unsupported("edge_mlp_bwd: hidden width above 512 is not built");
  }
  TFGNN_LAUNCH_CHECK();
  return 0;
}

static int launch_hidden_relu_src_bwd(const float* Xs, const float* Xt, const float* dA, const int* row_ptr_t,
                                      const int* tgt, int Vs, int L, int H, float* dXs, cudaStream_t st) {
  const int g = warp_grid((long long)L * Vs);
#define TFGNN_SRC_BWD(NV)                                                                                            \
  do {                                                                                                               \
    if (Xt) hidden_relu_src_bwd_kernel<NV, true><<<g, 256, 0, st>>>(Xs, Xt, dA, row_ptr_t, tgt, Vs, L, H, dXs);    \
    else hidden_relu_src_bwd_kernel<NV, false><<<g, 256, 0, st>>>(Xs, Xt, dA, row_ptr_t, tgt, Vs, L, H, dXs);      \
  } while (0)
  switch ((H + 127) / 128) {
    case 1: TFGNN_SRC_BWD(1); break;
    case 2: TFGNN_SRC_BWD(2); break;
    case 3: TFGNN_SRC_BWD(3); break;
    case 4: TFGNN_SRC_BWD(4); break;
    default: return unsupported("edge_mlp_bwd: hidden width above 512 is not built");
  }
#undef TFGNN_SRC_BWD
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn

extern "C" int tfgnn_b200_edge_mlp_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D,
                                       const float* const* mlp_weights, int32_t num_hidden_layers, int32_t H,
                                       uint32_t flags, int32_t aggregation, int32_t activation, const float* out,
                                       const float* grad_out, float* grad_h, float* const* grad_weights, void* stream) {
  // the configuration is judged from the scalar arguments alone, before any batch is read
  TFGNN_REQUIRE(D > 0 && H > 0, "D and H must be positive");
  TFGNN_REQUIRE(num_hidden_layers >= 0, "num_hidden_layers must be >= 0");
  TFGNN_REQUIRE(valid_act(activation) && valid_agg(aggregation), "unknown activation / aggregation code");
  if (num_hidden_layers != 1)
    return unsupported("edge_mlp_bwd differentiates one hidden layer (0: tfgnn_b200_rgcn_bwd; 2 or more are not built)");
  if (flags & TFGNN_FLAG_ACT_BEFORE_AGGREGATION)
    return unsupported("edge_mlp_bwd: activation-before-aggregation is not built yet");
  if (aggregation == TFGNN_AGG_MAX) return unsupported("edge_mlp_bwd: max aggregation is not built yet");
  if (D % 4 != 0 || H % 4 != 0) return unsupported("edge_mlp_bwd needs D and H to be multiples of 4");
  if (H > 512) return unsupported("edge_mlp_bwd: hidden width above 512 is not built");
  TFGNN_REQUIRE(b != nullptr && bt != nullptr, "batch / transposed batch is NULL");
  // V = owned target rows (of out / grad_out), Vs = rows of h and grad_h, lo = global id of local target 0
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L;
  if (int rc = check_backward_pair(b, bt)) return rc;
  TFGNN_REQUIRE(L == 0 || (mlp_weights && grad_weights), "weight / weight-gradient table is NULL");
  const bool use_target = flags & TFGNN_FLAG_USE_TARGET_STATE;   // U_l is then [2D, H]: rows [0,D) source, [D,2D) target
  const int KU = use_target ? 2 * D : D;                          // rows of U_l
  PtrTable us{}, w2{}, gw2{};
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(mlp_weights[2 * l] && mlp_weights[2 * l + 1] && grad_weights[2 * l] && grad_weights[2 * l + 1],
                  "a weight pointer is NULL");
    us.p[l] = mlp_weights[2 * l];
    w2.p[l] = mlp_weights[2 * l + 1];
    gw2.p[l] = grad_weights[2 * l + 1];
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0 || L == 0)   // no owned rows (an empty shard) or no edge types: zero contribution
    return zero_contribution({{grad_weights, L, (size_t)KU * H, 2}, {grad_weights + 1, L, (size_t)H * H, 2}}, grad_h,
                             (size_t)Vs * D, st);
  TFGNN_REQUIRE(h && out && grad_out, "NULL pointer");
  const float* h_tgt = h + (size_t)lo * D;   // rows of the owned targets (target-state input)
  const bool normalize = flags & TFGNN_FLAG_NORMALIZE_BY_NUM_INCOMING;
  const int LH = L * H;
  // 1. dZ = dOut * act'(out) * rn(v)
  PoolBuffer dz{st};
  int rc = begin_backward(b, bt, out, grad_out, H, activation, aggregation, st, dz, [&](float* z) {
    return edge_mlp_core(b, h, D, mlp_weights, 1, H, flags, aggregation, TFGNN_ACT_NONE, TFGNN_PATH_AUTO, z, H, st);
  });
  if (rc) return rc;
  PoolBuffer Xs{st}, Xt{st}, A{st}, cnt{st}, dXs{st}, Wp{st}, part{st};
  rc = Xs.alloc((size_t)Vs * LH * sizeof(float));
  if (!rc) rc = A.alloc((size_t)V * LH * sizeof(float));                              // A, then dA
  if (!rc) rc = Wp.alloc((size_t)(D > H ? D : H) * LH * sizeof(float));               // [D, LH] packs, then [LH, D]
  if (!rc) rc = dXs.alloc((size_t)Vs * LH * sizeof(float));
  if (!rc && use_target) rc = Xt.alloc((size_t)V * LH * sizeof(float));
  if (!rc && use_target) rc = cnt.alloc((size_t)V * LH * sizeof(float));              // cnt, then dXt
  if (!rc) {
    const size_t a = tn_partial_floats(V, LH, H), c = tn_partial_floats(Vs, D, H);
    rc = part.alloc((a > c ? a : c) * sizeof(float));
  }
  if (rc) return rc;

  // 2. Xs, Xt and A_l (+ cnt_l) recomputed with the forward's GEMMs and summation order
  GemmEpilogue none;
  rc = launch_pack_horizontal(us, L, 0, D, H, H, Wp.f(), LH, st);
  if (rc) return rc;
  rc = node_gemm(h, D, Wp.f(), LH, Xs.f(), LH, Vs, LH, D, none, TFGNN_PATH_AUTO, st);
  if (rc) return rc;
  if (use_target) {
    rc = launch_pack_horizontal(us, L, D, D, H, H, Wp.f(), LH, st);
    if (rc) return rc;
    rc = node_gemm(h_tgt, D, Wp.f(), LH, Xt.f(), LH, V, LH, D, none, TFGNN_PATH_AUTO, st);
    if (rc) return rc;
    rc = launch_hidden_relu_count(Xs.f(), Xt.f(), b->row_ptr, b->src_sorted, (int)V, L, H, normalize, A.f(), cnt.f(), st);
    if (rc) return rc;
  } else {
    EdgeReduceParams p;
    p.X = Xs.f(); p.ldx = LH; p.x_type_stride = H;
    p.row_ptr = b->row_ptr; p.src = b->src_sorted;
    p.out = A.f(); p.ldo = LH; p.out_type_stride = H;
    p.V = (int)V; p.L = L; p.C = H; p.normalize = normalize; p.hidden_relu = 1;
    rc = launch_edge_reduce(p, /*merged=*/false, st);
    if (rc) return rc;
  }
  // 3. dW2_l = A_l^T dZ
  rc = weight_grad(A.f(), LH, dz.f(), H, V, LH, H, part.f(), gw2, L, H, 0, st);
  if (rc) return rc;
  // 4. dA = dZ [W2_0; ..]^T (overwrites A), dA_l[v] *= s_{v,l}
  {
    PoolBuffer W2T{st};
    rc = W2T.alloc((size_t)LH * H * sizeof(float));
    if (!rc) rc = gemm_transposed(dz.f(), H, {w2, L, H, H}, W2T.f(), A.f(), LH, V, LH, none, st);
    if (rc) return rc;
  }
  if (normalize) {
    scale_by_type_kernel<<<grid_for(V * LH), 256, 0, st>>>(A.f(), LH, V, L, H, b->row_ptr);
    TFGNN_LAUNCH_CHECK();
  }
  // 5. dXs over the source-keyed CSR (on a shard: its owned transpose, every global source, local target ids);
  //    dXt = dA * cnt in place of cnt
  rc = launch_hidden_relu_src_bwd(Xs.f(), Xt.f(), A.f(), bt->row_ptr, bt->src_sorted, (int)Vs, L, H, dXs.f(), st);
  if (rc) return rc;
  if (use_target) {
    mul_inplace_kernel<<<grid_for(V * LH), 256, 0, st>>>(cnt.f(), A.f(), V * LH);
    TFGNN_LAUNCH_CHECK();
  }
  // 6. dU^s_l = h^T dXs_l over all Vs rows, dU^t_l = h_v^T dXt_l over the owned rows (rows [D, 2D) of U_l)
  for (int l = 0; l < L; ++l) {
    const PtrTable gu = one_table(grad_weights[2 * l]);
    rc = weight_grad(h, D, dXs.f() + (size_t)l * H, LH, Vs, D, H, part.f(), gu, 1, D, 0, st);
    if (rc) return rc;
    if (use_target) {
      rc = weight_grad(h_tgt, D, cnt.f() + (size_t)l * H, LH, V, D, H, part.f(), gu, 1, D, D, st);
      if (rc) return rc;
    }
  }
  if (!grad_h) return 0;
  // 7. grad_h = dXs [U^s_0^T; ..] (K = L*H), then the owned rows += dXt [U^t_0^T; ..]
  rc = gemm_transposed(dXs.f(), LH, {us, L, D, H, 1, 0, /*stacked=*/true}, Wp.f(), grad_h, D, Vs, D, none, st);
  if (rc || !use_target) return rc;
  GemmEpilogue acc;
  acc.accumulate = 1;
  return gemm_transposed(cnt.f(), LH, {us, L, D, H, 1, D, /*stacked=*/true}, Wp.f(), grad_h + (size_t)lo * D, D, V, D, acc,
                         st);
}

// =====================================================================================================================
// RGAT backward (rgat.py:91-163 through tfgnn_b200_rgat_fwd; edge-level kernels and their math in rgat.cu).  With
// P_l = h W_l, the score halves s_src, s_tgt of the forward and dZ = dOut * act':
//   1. dZ (gelu: the pre-activation from the forward's target walk with activation none)
//   2. P, s_src, s_tgt recomputed by the forward's rgat_tables: the forward's bits
//   3. target pass: m, den, g = dZ . o per (v, k) and ds_tgt [V, L*K]
//   4. source pass over the source-keyed CSR: dP [Vs, L*H] (messages and both score halves) and ds_src [Vs, L*K]
//   5. da_l = [sum_u ds_src P_l[u] | sum_v ds_tgt P_l[v]] per head (fixed row chunks, reduced in chunk order)
//   6. dW_l = h^T dP_l (TN, fixed 8192-row chunks),  7. grad_h = dP [W_0^T; ..]
// Every temporary is node-sized; nothing has a per-edge dimension and nothing uses float atomics.  On a shard dP, ds_src and
// grad_h cover every source (bt is the owned transpose), the target pass and ds_tgt the owned rows.
// =====================================================================================================================
extern "C" int tfgnn_b200_rgat_bwd(tfgnn_batch_t* b, tfgnn_batch_t* bt, const float* h, int32_t D, const float* const* W,
                                   const float* const* attention, int32_t H, int32_t num_heads, int32_t activation,
                                   int32_t path, const float* out, const float* grad_out, float* grad_h,
                                   float* const* grad_W, float* const* grad_attention, void* stream) {
  // the configuration is judged from the scalar arguments alone, before any batch is read
  TFGNN_REQUIRE(D > 0 && H > 0 && num_heads > 0, "D, H and num_heads must be positive");
  TFGNN_REQUIRE(H % num_heads == 0, "hidden_dim must be divisible by num_heads (rgat.py:72)");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  const int K = num_heads, d = H / num_heads;
  if (D % 4 != 0 || d % 4 != 0) return unsupported("rgat_bwd needs D and hidden_dim / num_heads to be multiples of 4");
  if (H > 512) return unsupported("rgat_bwd: hidden_dim above 512 is not built");
  if (path == TFGNN_PATH_ATOMIC) return unsupported("rgat_bwd: TFGNN_PATH_ATOMIC is not available for RGAT");
  TFGNN_REQUIRE(b != nullptr && bt != nullptr, "batch / transposed batch is NULL");
  // V = owned target rows (of out / grad_out), Vs = rows of h and grad_h, lo = global id of local target 0
  const long long V = b->V, Vs = b->V_src, lo = b->tgt_off;
  const int L = b->L;
  if (int rc = check_backward_pair(b, bt)) return rc;
  TFGNN_REQUIRE(L == 0 || (W && attention && grad_W && grad_attention), "weight / weight-gradient table is NULL");
  PtrTable wt{}, at{}, gat{};
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(W[l] && attention[l] && grad_W[l] && grad_attention[l], "a weight pointer is NULL");
    wt.p[l] = W[l];
    at.p[l] = attention[l];
    gat.p[l] = grad_attention[l];
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0 || L == 0)   // no owned rows (an empty shard) or no edge types: zero contribution
    return zero_contribution({{grad_W, L, (size_t)D * H}, {grad_attention, L, (size_t)2 * H}}, grad_h, (size_t)Vs * D, st);
  TFGNN_REQUIRE(h && out && grad_out, "NULL pointer");
  const int LH = L * H, LK = L * K;
  // 1. dZ = dOut * act'(out)
  PoolBuffer dz{st};
  int rc = begin_backward(b, bt, out, grad_out, H, activation, TFGNN_AGG_SUM, st, dz, [&](float* z) {
    PoolBuffer P{st}, ss{st}, stt{st};
    const int r = rgat_tables(b, h, D, wt, at, H, K, path, P, ss, stt, st);
    return r ? r : launch_rgat_aggregate(b, P.f(), ss.f(), stt.f(), K, d, TFGNN_ACT_NONE, z, st);
  });
  if (rc) return rc;
  // 2. the forward's tables
  PoolBuffer P{st}, ss{st}, stt{st};
  rc = rgat_tables(b, h, D, wt, at, H, K, path, P, ss, stt, st);
  if (rc) return rc;
  PoolBuffer stat{st}, ds_tgt{st}, dP{st}, ds_src{st};
  rc = stat.alloc((size_t)V * 3 * K * sizeof(float));
  if (!rc) rc = ds_tgt.alloc((size_t)V * LK * sizeof(float));
  if (!rc) rc = dP.alloc((size_t)Vs * LH * sizeof(float));
  if (!rc) rc = ds_src.alloc((size_t)Vs * LK * sizeof(float));
  if (rc) return rc;
  // 3., 4. target pass, source pass
  rc = launch_rgat_target_pass(b, P.f(), ss.f(), stt.f(), K, d, dz.f(), stat.f(), ds_tgt.f(), st);
  if (rc) return rc;
  rc = launch_rgat_source_pass(b, bt, P.f(), ss.f(), stt.f(), at, K, d, dz.f(), stat.f(), ds_tgt.f(), dP.f(), ds_src.f(),
                               st);
  if (rc) return rc;
  // 5. attention gradients: the source half over all Vs rows, the target half over the owned rows
  rc = launch_rgat_attention_grad(ds_src.f(), P.f(), Vs, L, K, d, gat, 0, st);
  if (rc) return rc;
  rc = launch_rgat_attention_grad(ds_tgt.f(), P.f() + (size_t)lo * LH, V, L, K, d, gat, 1, st);
  if (rc) return rc;
  // 6. dW_l = h^T dP_l over all Vs rows
  {
    PoolBuffer part{st};
    rc = part.alloc(tn_partial_floats(Vs, D, H) * sizeof(float));
    for (int l = 0; l < L && !rc; ++l)
      rc = weight_grad(h, D, dP.f() + (size_t)l * H, LH, Vs, D, H, part.f(), one_table(grad_W[l]), 1, D, 0, st);
    if (rc) return rc;
  }
  if (!grad_h) return 0;
  // 7. grad_h = dP [W_0^T; ..] (K = L*H)
  PoolBuffer WT{st};
  rc = WT.alloc((size_t)LH * D * sizeof(float));
  return rc ? rc : gemm_transposed(dP.f(), LH, {wt, L, D, H, 1, 0, /*stacked=*/true}, WT.f(), grad_h, D, Vs, D,
                                   GemmEpilogue{}, st);
}

// =====================================================================================================================
// Node-level glue of GNN._internal_call under training (gnn.py:279-327): backward of the bias-free / biased Dense layers,
// LayerNormalization, and the Philox dropout shared by forward and backward.  The reference gets all of these from
// tf.GradientTape (models/graph_task_model.py:338-365).
// =====================================================================================================================
namespace tfgnn {

// LayerNormalization backward, one warp per row:
//   xhat = (x - mean) * rstd;  dxhat = g * gamma;
//   dx = rstd * (dxhat - mean(dxhat) - xhat * mean(dxhat * xhat));   t[v,c] = g * xhat  (column-summed into dgamma)
__global__ void layer_norm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                      const float* __restrict__ g, long long V, int H, float eps,
                                      float* __restrict__ dx, float* __restrict__ t) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= V) return;
  const float* xr = x + row * H;
  const float* gr = g + row * H;
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
  const float rstd = rsqrtf(q / (float)H + eps);
  float a = 0.f, b = 0.f;   // sum dxhat, sum dxhat * xhat
  for (int c = lane; c < H; c += 32) {
    const float xhat = (xr[c] - mean) * rstd;
    const float dxh = gr[c] * gamma[c];
    a += dxh;
    b += dxh * xhat;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  a /= (float)H;
  b /= (float)H;
  for (int c = lane; c < H; c += 32) {
    const float xhat = (xr[c] - mean) * rstd;
    const float dxh = gr[c] * gamma[c];
    if (dx) dx[row * H + c] = rstd * (dxh - a - xhat * b);
    t[row * H + c] = gr[c] * xhat;
  }
}

// Philox4x32-10 (Salmon et al. 2011), the counter-based generator TensorFlow's stateless random ops use as well.
// One counter value yields 4 uniform 32-bit words: element i takes word i & 3 of counter i >> 2, so the mask of an
// element depends only on (seed, offset, i): the backward pass regenerates it instead of storing it.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// tf.nn.dropout(x, rate): keep with probability 1 - rate, scale kept values by 1 / (1 - rate)   (gnn.py:285-289)
// x[i] is element first + i of the masked table: its mask is word (first + i) % 4 of Philox counter offset + (first + i) / 4.
__global__ void dropout_kernel(const float* __restrict__ x, long long n, float rate, unsigned long long seed,
                               unsigned long long offset, long long first, float* __restrict__ out) {
  const float scale = 1.0f / (1.0f - rate);
  const long long g0 = first >> 2;
  const long long groups = ((first + n + 3) >> 2) - g0;
  for (long long gi = (long long)blockIdx.x * blockDim.x + threadIdx.x; gi < groups;
       gi += (long long)gridDim.x * blockDim.x) {
    const unsigned long long c = (unsigned long long)(g0 + gi) + offset;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), 0u, 0u),
                                  make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = (g0 + gi) * 4 + j - first;
      if (i >= 0 && i < n) {
        const float u = (float)(w[j] >> 8) * (1.0f / 16777216.0f);   // uniform in [0, 1)
        out[i] = u >= rate ? x[i] * scale : 0.0f;
      }
    }
  }
}

__global__ void axpby_kernel(const float* __restrict__ a, float alpha, const float* __restrict__ b, float beta,
                             long long n, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = b ? alpha * a[i] + beta * b[i] : alpha * a[i];
}

}  // namespace tfgnn

// Backward of out = act(x W + bias): grad_x = dZ W^T (tensor-core GEMM), grad_W = x^T dZ (TN GEMM, fixed-order partials),
// grad_bias = column sums of dZ, dZ = grad_out * act'.  `out` is the saved forward output.
extern "C" int tfgnn_b200_dense_bwd(const float* x, const float* W, const float* bias, const float* out,
                                    const float* grad_out, int64_t V, int32_t K, int32_t N, int32_t activation,
                                    float* grad_x, float* grad_W, float* grad_bias, void* stream) {
  TFGNN_REQUIRE(V >= 0 && K > 0 && N > 0, "bad dense shape");
  TFGNN_REQUIRE(valid_act(activation), "unknown activation code");
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0) {
    if (grad_W) TFGNN_CUDA(cudaMemsetAsync(grad_W, 0, (size_t)K * N * sizeof(float), st));
    if (grad_bias) TFGNN_CUDA(cudaMemsetAsync(grad_bias, 0, (size_t)N * sizeof(float), st));
    return 0;
  }
  TFGNN_REQUIRE(x && W && out && grad_out, "NULL pointer");
  PoolBuffer dz{st}, pre{st};
  int rc = dz.alloc((size_t)V * N * sizeof(float));
  if (rc) return rc;
  const float* y = out;
  if (activation == TFGNN_ACT_GELU) {   // derivative needs the pre-activation: recompute x W + bias
    rc = pre.alloc((size_t)V * N * sizeof(float));
    if (!rc) rc = tfgnn_b200_dense_bias_fwd(x, W, bias, pre.f(), V, K, N, TFGNN_ACT_NONE, TFGNN_PATH_AUTO, stream);
    if (rc) return rc;
    y = pre.f();
  }
  rc = tfgnn_b200_activation_bwd(y, grad_out, V * N, activation, dz.f(), stream);
  if (rc) return rc;
  if (grad_W) {
    PoolBuffer part{st};
    rc = part.alloc(tn_partial_floats(V, K, N) * sizeof(float));
    if (!rc) rc = weight_grad(x, K, dz.f(), N, V, K, N, part.f(), one_table(grad_W), 1, K, 0, st);
    if (rc) return rc;
  }
  if (grad_bias) {
    rc = column_sums(dz.f(), V, N, grad_bias, nullptr, st);
    if (rc) return rc;
  }
  if (!grad_x) return 0;
  PoolBuffer wT{st};
  rc = wT.alloc((size_t)N * K * sizeof(float));
  if (rc) return rc;
  return gemm_transposed(dz.f(), N, {one_table(W), 1, K, N}, wT.f(), grad_x, K, V, K, GemmEpilogue{}, st);
}

extern "C" int tfgnn_b200_layer_norm_bwd(const float* x, const float* gamma, const float* grad_out, int64_t V, int32_t H,
                                         float epsilon, float* grad_x, float* grad_gamma, float* grad_beta,
                                         void* stream) {
  TFGNN_REQUIRE(V >= 0 && H > 0, "bad layer_norm shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0) {
    if (grad_gamma) TFGNN_CUDA(cudaMemsetAsync(grad_gamma, 0, (size_t)H * sizeof(float), st));
    if (grad_beta) TFGNN_CUDA(cudaMemsetAsync(grad_beta, 0, (size_t)H * sizeof(float), st));
    return 0;
  }
  TFGNN_REQUIRE(x && gamma && grad_out, "NULL pointer");
  PoolBuffer t{st};
  int rc = t.alloc((size_t)V * H * sizeof(float));
  if (rc) return rc;
  layer_norm_bwd_kernel<<<ceil_div(V * 32, 256), 256, 0, st>>>(x, gamma, grad_out, V, H, epsilon, grad_x, t.f());
  TFGNN_LAUNCH_CHECK();
  if (grad_gamma) {
    rc = column_sums(t.f(), V, H, grad_gamma, nullptr, st);
    if (rc) return rc;
  }
  return grad_beta ? column_sums(grad_out, V, H, grad_beta, nullptr, st) : 0;
}

// tf.nn.dropout (gnn.py:285-289, graph_global_exchange.py:98-101).  The mask is a pure function of (seed, offset, element
// index), so the backward pass calls the same entry on the incoming gradient.
extern "C" int tfgnn_b200_dropout(const float* x, int64_t n, float rate, uint64_t seed, uint64_t offset, float* out,
                                  void* stream) {
  TFGNN_REQUIRE(n >= 0 && rate >= 0.0f && rate < 1.0f, "dropout rate must lie in [0, 1)");
  if (n == 0) return 0;
  TFGNN_REQUIRE(x && out, "NULL pointer");
  dropout_kernel<<<grid_for((n + 3) / 4), 256, 0, (cudaStream_t)stream>>>(x, n, rate, seed, offset, 0, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

// The same masks for a slice of a larger table: x is elements [first_element, first_element + n) of the table a call of
// tfgnn_b200_dropout with the same (seed, offset) would mask (a target-range shard's rows of a [V, H] table).
extern "C" int tfgnn_b200_dropout_at(const float* x, int64_t n, float rate, uint64_t seed, uint64_t offset,
                                     int64_t first_element, float* out, void* stream) {
  TFGNN_REQUIRE(n >= 0 && rate >= 0.0f && rate < 1.0f, "dropout rate must lie in [0, 1)");
  TFGNN_REQUIRE(first_element >= 0, "dropout_at: first_element must not be negative");
  if (n == 0) return 0;
  TFGNN_REQUIRE(x && out, "NULL pointer");
  dropout_kernel<<<grid_for((first_element % 4 + n + 3) / 4), 256, 0, (cudaStream_t)stream>>>(x, n, rate, seed, offset,
                                                                                               first_element, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

extern "C" int tfgnn_b200_axpby(const float* a, float alpha, const float* b, float beta, int64_t n, float* out,
                                void* stream) {
  TFGNN_REQUIRE(n >= 0, "negative size");
  if (n == 0) return 0;
  TFGNN_REQUIRE(a && out, "NULL pointer");
  axpby_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(a, alpha, b, beta, n, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}
