// Edge-level kernels: gather source-node rows along the (type,target)-sorted CSR and reduce
// them per target.  HBM-bound: one 8 B index pair (amortised into the 4 B sorted source id) and
// 4*C bytes of node-table row per edge; no [E,D] gather, [E,H] message or [M,H] concat buffer
// is ever materialised (the reference materialises all three: message_passing.py:197-206,
// gnn_edge_mlp.py:100, message_passing.py:166-167).
//
// One warp owns one segment (PER_TYPE mode: segment (l,v) -> out[v, l*stride + :]) or one
// target node (MERGED mode: all L segments of v reduced into out[v, :]), so the reduction is a
// register accumulation in CSR order: no atomics, run-to-run deterministic.
#include <cstdlib>

#include "edge_reduce.cuh"

namespace tfgnn {

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int NV>
struct RowAcc {
  float4 v[NV];
};

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4_max(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float4 f4_scale(float4 a, float s) {
  return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}
__device__ __forceinline__ float4 f4_fill(float s) { return make_float4(s, s, s, s); }

// Per-edge message transform on pre-projected rows (everything that is NOT a matmul in
// gnn_edge_mlp.py:84-107 / gnn_film.py:99-107 / message_passing.py:169-170).  pre() is the message before the activation,
// act() the activation; the backward's edge_grad_kernel calls the two halves so that it sees the forward's bits.
struct EdgeFn {
  float4 t, g, b;  // target-side additive term, FiLM gamma / beta for this (v,l) and column group
  float scale;
  bool has_t, hidden_relu, scale_per_edge, film;
  int edge_act;
  __device__ __forceinline__ float4 pre(float4 x) const {
    if (has_t) x = f4_add(x, t);
    if (hidden_relu) x = f4_max(x, f4_fill(0.f));
    if (scale_per_edge) x = f4_scale(x, scale);
    if (film) x = make_float4(g.x * x.x + b.x, g.y * x.y + b.y, g.z * x.z + b.z, g.w * x.w + b.w);
    return x;
  }
  __device__ __forceinline__ float4 act(float4 x) const {
    if (edge_act != TFGNN_ACT_NONE)
      x = make_float4(apply_act(x.x, edge_act), apply_act(x.y, edge_act), apply_act(x.z, edge_act),
                      apply_act(x.w, edge_act));
    return x;
  }
  __device__ __forceinline__ float4 operator()(float4 x) const { return act(pre(x)); }
};

// 1/(c_{v,l}+eps) of gnn_edge_mlp.py:102-106, or 1
__device__ __forceinline__ float segment_scale(int cnt, int normalize) {
  return normalize ? 1.0f / ((float)cnt + kSmallNumber) : 1.0f;
}

// Running maximum with its tie count: n counts the messages equal to the maximum so far (a larger message restarts it),
// so after the last message n = #{e : y_e == max} per column, the count of tf.math.unsorted_segment_max's gradient.
__device__ __forceinline__ float tie_step(float n, float acc, float y) {
  return y > acc ? 1.f : (y == acc ? n + 1.f : n);
}
__device__ __forceinline__ float4 f4_tie_step(float4 n, float4 acc, float4 y) {
  return make_float4(tie_step(n.x, acc.x, y.x), tie_step(n.y, acc.y, y.y), tie_step(n.z, acc.z, y.z),
                     tie_step(n.w, acc.w, y.w));
}

// NV = float4 column groups per lane (C <= 128*NV).  PLAIN: identity message + sum, scale at end.
// U = edges loaded per round (loads in flight per lane = U*NV).  The lean PLAIN variant trades unroll
// depth for occupancy (<= 40 registers -> 6 CTAs/SM): the gather is bound by the number of independent
// row_ptr -> index -> row dependency chains in flight, i.e. by resident warps, not by loads per warp.
// TIES (MERGED max only): the tie count of every (v, c) goes to p.ties, taken along the same running maximum.
template <int NV, bool MERGED, bool PLAIN, int U = 4, int MINB = 1, bool TIES = false>
__global__ void __launch_bounds__(256, MINB) edge_reduce_kernel(const EdgeReduceParams p) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long warp_stride = ((long long)gridDim.x * blockDim.x) >> 5;
  const int vcount = p.v_count;
  const long long num_items = MERGED ? (long long)vcount : (long long)p.L * vcount;
  const int C4 = p.C >> 2;
  const bool use_max = (!PLAIN) && p.reduce_max;
  for (long long item = warp_global; item < num_items; item += warp_stride) {
  int l_first, l_last, v;
  if (MERGED) {
    v = p.v_begin + (int)item;
    l_first = 0;
    l_last = p.L;
  } else {
    l_first = (int)(item / vcount);
    l_last = l_first + 1;
    v = p.v_begin + (int)(item - (long long)l_first * vcount);
  }
  float4 acc[NV], ties[TIES ? NV : 1];
#pragma unroll
  for (int j = 0; j < NV; ++j) acc[j] = f4_fill(use_max ? kLowestFloat : 0.f);
  if (TIES) {
#pragma unroll
    for (int j = 0; j < NV; ++j) ties[j] = f4_fill(0.f);
  }
  int total_cnt = 0;


  for (int l = l_first; l < l_last; ++l) {
    const long long seg = (long long)l * p.V + v;
    const int beg = __ldg(p.row_ptr + seg), end = __ldg(p.row_ptr + seg + 1);
    const int cnt = end - beg;
    total_cnt += cnt;
    const float scale = segment_scale(cnt, p.normalize);
    const float* __restrict__ xbase = p.X + (long long)l * p.x_type_stride;
    EdgeFn fn[NV];
    if (!PLAIN) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const int c4 = lane + 32 * j;
        fn[j].has_t = p.T != nullptr;
        fn[j].hidden_relu = p.hidden_relu;
        fn[j].film = p.G != nullptr;
        fn[j].edge_act = p.edge_act;
        fn[j].scale = scale;
        fn[j].scale_per_edge = p.normalize && (p.G != nullptr || p.edge_act != TFGNN_ACT_NONE || use_max);
        fn[j].t = fn[j].g = fn[j].b = f4_fill(0.f);
        if (c4 < C4 && cnt > 0) {
          if (p.T) fn[j].t = ldg_f4(p.T + (long long)v * p.ldt + (long long)l * p.t_type_stride + 4 * c4);
          if (p.G) {
            const float* gp = p.G + (long long)v * p.ldg + (long long)l * p.g_type_stride + 4 * c4;
            fn[j].g = ldg_f4(gp);
            fn[j].b = ldg_f4(gp + p.beta_off);
          }
        }
      }
    }
    float4 part[NV];  // per-type partial (sum mode) so the end-of-segment scale is per type
#pragma unroll
    for (int j = 0; j < NV; ++j) part[j] = f4_fill(0.f);

    for (int base = beg; base < end; base += 32) {
      const int n = min(32, end - base);
      const int my_src = lane < n ? __ldg(p.src + base + lane) : 0;
      int e = 0;
      for (; e + U <= n; e += U) {
        float4 r[U][NV];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int s = __shfl_sync(0xffffffffu, my_src, e + u);
          const float* row = xbase + (long long)s * p.ldx;
#pragma unroll
          for (int j = 0; j < NV; ++j) {
            const int c4 = lane + 32 * j;
            r[u][j] = c4 < C4 ? ldg_f4(row + 4 * c4) : f4_fill(0.f);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int j = 0; j < NV; ++j) {
            if (PLAIN) {
              part[j] = f4_add(part[j], r[u][j]);
            } else {
              float4 y = fn[j](r[u][j]);
              if (TIES) ties[j] = f4_tie_step(ties[j], acc[j], y);
              if (use_max) acc[j] = f4_max(acc[j], y);
              else part[j] = f4_add(part[j], y);
            }
          }
      }
      for (; e < n; ++e) {
        const int s = __shfl_sync(0xffffffffu, my_src, e);
        const float* row = xbase + (long long)s * p.ldx;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const int c4 = lane + 32 * j;
          float4 x = c4 < C4 ? ldg_f4(row + 4 * c4) : f4_fill(0.f);
          if (PLAIN) {
            part[j] = f4_add(part[j], x);
          } else {
            float4 y = fn[j](x);
            if (TIES) ties[j] = f4_tie_step(ties[j], acc[j], y);
            if (use_max) acc[j] = f4_max(acc[j], y);
            else part[j] = f4_add(part[j], y);
          }
        }
      }
    }
    if (!use_max) {
      const bool scale_at_end = p.normalize && (PLAIN || !fn[0].scale_per_edge);
#pragma unroll
      for (int j = 0; j < NV; ++j)
        acc[j] = f4_add(acc[j], scale_at_end ? f4_scale(part[j], scale) : part[j]);
    }
  }

  // epilogue
  float rn = 1.0f;
  bool divide = false;
  if (MERGED && !PLAIN) {
    if (p.row_norm == 1) { rn = (float)max(total_cnt, 1); divide = true; }
    else if (p.row_norm == 2) { rn = sqrtf((float)max(total_cnt, 1)); divide = true; }
  }
  float* orow = p.out + (long long)(v - p.v_begin) * p.ldo + (MERGED ? 0 : (long long)l_first * p.out_type_stride);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int c4 = lane + 32 * j;
    if (c4 < C4) {
      float4 y = acc[j];
      if (divide) y = make_float4(y.x / rn, y.y / rn, y.z / rn, y.w / rn);
      if (!PLAIN && p.final_act != TFGNN_ACT_NONE)
        y = make_float4(apply_act(y.x, p.final_act), apply_act(y.y, p.final_act),
                        apply_act(y.z, p.final_act), apply_act(y.w, p.final_act));
      *reinterpret_cast<float4*>(orow + 4 * c4) = y;
      if (TIES) *reinterpret_cast<float4*>(p.ties + (long long)(v - p.v_begin) * p.ldo + 4 * c4) = ties[j];
    }
  }
  }  // item loop
}

// Scalar fallback for column counts / leading dimensions that are not multiples of 4 (doctest
// sizes such as D=3, H=7): one thread per (item, column).  Same semantics, no vector loads.
template <bool MERGED>
__global__ void edge_reduce_scalar_kernel(const EdgeReduceParams p) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long num_items = MERGED ? (long long)p.v_count : (long long)p.L * p.v_count;
  if (idx >= num_items * p.C) return;
  const long long item = idx / p.C;
  const int c = (int)(idx - item * p.C);
  int l_first, l_last, v;
  if (MERGED) { v = p.v_begin + (int)item; l_first = 0; l_last = p.L; }
  else { l_first = (int)(item / p.v_count); l_last = l_first + 1; v = p.v_begin + (int)(item - (long long)l_first * p.v_count); }
  const bool use_max = p.reduce_max;
  float acc = use_max ? kLowestFloat : 0.f;
  int total_cnt = 0;
  for (int l = l_first; l < l_last; ++l) {
    const long long seg = (long long)l * p.V + v;
    const int beg = p.row_ptr[seg], end = p.row_ptr[seg + 1];
    const int cnt = end - beg;
    total_cnt += cnt;
    const float scale = p.normalize ? 1.0f / ((float)cnt + kSmallNumber) : 1.0f;
    const bool film = p.G != nullptr;
    const bool scale_per_edge = p.normalize && (film || p.edge_act != TFGNN_ACT_NONE || use_max);
    float t = 0.f, g = 0.f, b = 0.f;
    if (cnt > 0) {
      if (p.T) t = p.T[(long long)v * p.ldt + (long long)l * p.t_type_stride + c];
      if (film) {
        const float* gp = p.G + (long long)v * p.ldg + (long long)l * p.g_type_stride + c;
        g = gp[0];
        b = gp[p.beta_off];
      }
    }
    float part = 0.f;
    for (int e = beg; e < end; ++e) {
      float x = p.X[(long long)p.src[e] * p.ldx + (long long)l * p.x_type_stride + c];
      if (p.T) x += t;
      if (p.hidden_relu) x = fmaxf(x, 0.f);
      if (scale_per_edge) x *= scale;
      if (film) x = g * x + b;
      x = apply_act(x, p.edge_act);
      if (use_max) acc = fmaxf(acc, x);
      else part += x;
    }
    if (!use_max) acc += (p.normalize && !scale_per_edge) ? part * scale : part;
  }
  if (MERGED) {
    if (p.row_norm == 1) acc = acc / (float)max(total_cnt, 1);
    else if (p.row_norm == 2) acc = acc / sqrtf((float)max(total_cnt, 1));
  }
  acc = apply_act(acc, p.final_act);
  p.out[(long long)(v - p.v_begin) * p.ldo + (MERGED ? 0 : (long long)l_first * p.out_type_stride) + c] = acc;
}

// Target-state term of a 0-hidden-layer edge MLP with use_target_state_as_input
// (gnn_edge_mlp.py:93-98): sum_e (h_v W^t) / (c+eps) = (c/(c+eps)) * h_v W^t, so the per-(v,l)
// input row of the node-level contraction is coeff(v,l) * h_v.
// Type l reads columns [l*in_stride, l*in_stride + D) of h (in_stride 0: every type reads the same row).
__global__ void target_term_kernel(const float* __restrict__ h, int ldh, const int* __restrict__ row_ptr,
                                   int V, int L, int D, int normalize, float* __restrict__ out, int ldo,
                                   int col0, int in_stride) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)V * L * D;
  if (idx >= total) return;
  const int c = (int)(idx % D);
  const long long vl = idx / D;
  const int l = (int)(vl % L);
  const int v = (int)(vl / L);
  const long long seg = (long long)l * V + v;
  const float cnt = (float)(row_ptr[seg + 1] - row_ptr[seg]);
  const float coeff = normalize ? cnt * (1.0f / (cnt + kSmallNumber)) : cnt;
  out[(long long)v * ldo + col0 + (long long)l * D + c] = coeff * h[(long long)v * ldh + (long long)l * in_stride + c];
}

// float4 version (D, ldh, ldo, col0 multiples of 4, aligned bases): one warp per node, the node's row is read ONCE and
// written L times (the scalar kernel above re-read it L times through a div/mod per element: 17 ms for 15 GB at the
// GNN-FiLM 1/8 shard, 0.9 TB/s).
__global__ void __launch_bounds__(256) target_term_vec_kernel(const float* __restrict__ h, int ldh,
                                                              const int* __restrict__ row_ptr, int V, int L, int D,
                                                              int normalize, float* __restrict__ out, int ldo, int col0,
                                                              int in_stride) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int C4 = D >> 2;
  for (long long v = warp; v < V; v += nwarps) {
    const float* hr = h + v * ldh;
    float* orow = out + v * ldo + col0;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      float4 x = ldg_f4(hr + 4 * c4);
      for (int l = 0; l < L; ++l) {
        if (in_stride && l) x = ldg_f4(hr + (long long)l * in_stride + 4 * c4);
        const long long seg = (long long)l * V + v;
        const float cnt = (float)(__ldg(row_ptr + seg + 1) - __ldg(row_ptr + seg));
        const float coeff = normalize ? cnt * (1.0f / (cnt + kSmallNumber)) : cnt;
        *reinterpret_cast<float4*>(orow + (long long)l * D + 4 * c4) =
            make_float4(coeff * x.x, coeff * x.y, coeff * x.z, coeff * x.w);
      }
    }
  }
}

// Backward of the merged transform-then-aggregate reduce f (DESIGN.md §6).  Per edge e = (u -> v) of type l, with
// x_e = EdgeFn::pre(P_l[u]) = (P_l[u] + T_l[v]) s and y_e = EdgeFn::act(x_e), computed by the forward's code:
//   w_e = dZ[v] * [y_e == z[v]] (max only) * act'(x_e) (activation before aggregation only) * s
// KEY_SRC: out_l[u] = sum of w_e over the edges LEAVING u (the source-keyed CSR: segment (l, u), values = target rows) = dP_l
// else:    out_l[v] = sum of w_e over the edges INTO v (f's CSR: segment (l, v), values = source rows)            = dT_l
// One warp per segment, lanes over float4 column groups, edges in CSR order: no atomics, deterministic.  A segment is one
// warp's serial work, however many edges it has.  Segments without edges get zero rows.
struct EdgeGradArgs {
  EdgeReduceParams f;
  const float* z;    // [f.V, f.C] maximum per target (max only, else NULL)
  const float* dz;   // [f.V, f.C]
  const int* row_ptr;
  const int* idx;
  int Vk;            // segments per type of the walked CSR
  float* out;        // [Vk, f.L * f.C]
};

__device__ __forceinline__ float edge_weight(float x, float y, float dz, float z, bool use_max, int edge_act, float s) {
  float w = (use_max && y != z) ? 0.f : dz;
  if (edge_act != TFGNN_ACT_NONE)
    w *= edge_act == TFGNN_ACT_GELU ? gelu_grad_from_input(x) : act_grad_from_output(y, edge_act);
  return w * s;
}

template <int NV>
__device__ __forceinline__ void load_target_side(const EdgeGradArgs& a, int l, int v, int cnt, EdgeFn (&fn)[NV],
                                                 float4 (&dz)[NV], float4 (&z)[NV]) {
  const int lane = threadIdx.x & 31, C4 = a.f.C >> 2;
  const float s = segment_scale(cnt, a.f.normalize);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int c4 = lane + 32 * j;
    fn[j].scale = s;
    if (c4 >= C4) continue;
    if (a.f.T) fn[j].t = ldg_f4(a.f.T + (long long)v * a.f.ldt + (long long)l * a.f.t_type_stride + 4 * c4);
    dz[j] = ldg_f4(a.dz + (long long)v * a.f.C + 4 * c4);
    if (a.z) z[j] = ldg_f4(a.z + (long long)v * a.f.C + 4 * c4);
  }
}

template <int NV, bool KEY_SRC>
__global__ void __launch_bounds__(256) edge_grad_kernel(const EdgeGradArgs a) {
  const EdgeReduceParams& f = a.f;
  const int lane = threadIdx.x & 31;
  const int C4 = f.C >> 2;
  const long long ldo = (long long)f.L * f.C;
  const long long items = (long long)f.L * a.Vk;
  const bool use_max = a.z != nullptr;
  for (long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < items;
       item += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int l = (int)(item / a.Vk), k = (int)(item - (long long)l * a.Vk);
    const int beg = __ldg(a.row_ptr + item), end = __ldg(a.row_ptr + item + 1);
    const float* __restrict__ xbase = f.X + (long long)l * f.x_type_stride;
    EdgeFn fn[NV];
    float4 key_row[NV], dz[NV], z[NV], acc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      fn[j].has_t = f.T != nullptr;
      fn[j].hidden_relu = false;
      fn[j].film = false;
      fn[j].edge_act = f.edge_act;
      fn[j].scale_per_edge = f.normalize;
      fn[j].scale = 1.f;
      fn[j].t = fn[j].g = fn[j].b = key_row[j] = dz[j] = z[j] = acc[j] = f4_fill(0.f);
    }
    if (end > beg) {
      if (KEY_SRC) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const int c4 = lane + 32 * j;
          if (c4 < C4) key_row[j] = ldg_f4(xbase + (long long)k * f.ldx + 4 * c4);
        }
      } else {
        load_target_side<NV>(a, l, k, end - beg, fn, dz, z);
      }
    }
    for (int base = beg; base < end; base += 32) {
      const int m = min(32, end - base);
      const int my_other = lane < m ? __ldg(a.idx + base + lane) : 0;
#pragma unroll 1
      for (int e = 0; e < m; ++e) {
        const int o = __shfl_sync(0xffffffffu, my_other, e);
        if (KEY_SRC) {
          const long long seg = (long long)l * f.V + o;
          load_target_side<NV>(a, l, o, __ldg(f.row_ptr + seg + 1) - __ldg(f.row_ptr + seg), fn, dz, z);
        }
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const int c4 = lane + 32 * j;
          if (c4 >= C4) continue;
          const float4 r = KEY_SRC ? key_row[j] : ldg_f4(xbase + (long long)o * f.ldx + 4 * c4);
          const float4 x = fn[j].pre(r), y = fn[j].act(x);
          const float s = fn[j].scale;
          acc[j].x += edge_weight(x.x, y.x, dz[j].x, z[j].x, use_max, f.edge_act, s);
          acc[j].y += edge_weight(x.y, y.y, dz[j].y, z[j].y, use_max, f.edge_act, s);
          acc[j].z += edge_weight(x.z, y.z, dz[j].z, z[j].z, use_max, f.edge_act, s);
          acc[j].w += edge_weight(x.w, y.w, dz[j].w, z[j].w, use_max, f.edge_act, s);
        }
      }
    }
    float* orow = a.out + (long long)k * ldo + (long long)l * f.C;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c4 = lane + 32 * j;
      if (c4 < C4) *reinterpret_cast<float4*>(orow + 4 * c4) = acc[j];
    }
  }
}

// Per-edge red.global.add path (TFGNN_PATH_ATOMIC): the stock-TF-GPU formulation
// (UnsortedSegmentSum = atomicAdd).  Kept as the measured alternative to the CSR path.
__global__ void edge_scatter_atomic_kernel(const int2* __restrict__ edges, long long E, int l, int V,
                                           const float* __restrict__ X, int ldx, int C,
                                           const int* __restrict__ row_ptr, int normalize,
                                           float* __restrict__ out, int ldo, int col0) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long num_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int C4 = C >> 2;
  for (long long e = warp; e < E; e += num_warps) {
    const int2 st = __ldg(edges + e);
    if ((unsigned)st.x >= (unsigned)V || (unsigned)st.y >= (unsigned)V) continue;
    const long long seg = (long long)l * V + st.y;
    const float scale = normalize ? 1.0f / ((float)(__ldg(row_ptr + seg + 1) - __ldg(row_ptr + seg)) + kSmallNumber) : 1.0f;
    const float* row = X + (long long)st.x * ldx;
    float* orow = out + (long long)st.y * ldo + col0;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      float4 x = f4_scale(ldg_f4(row + 4 * c4), scale);
      atomicAdd(reinterpret_cast<float4*>(orow + 4 * c4), x);  // red.global.add.v4.f32 (sm_90+)
    }
  }
}


int launch_edge_reduce(const EdgeReduceParams& p_in, bool merged, cudaStream_t st, int max_blocks) {
  EdgeReduceParams p = p_in;
  if (p.v_count <= 0) {  // full range
    p.v_begin = 0;
    p.v_count = p.V;
  }
  const long long items = merged ? (long long)p.v_count : (long long)p.L * p.v_count;
  if (items == 0 || p.C == 0) return 0;
  const bool plain = !merged && !p.T && !p.G && !p.hidden_relu && p.edge_act == TFGNN_ACT_NONE &&
                     !p.reduce_max && p.final_act == TFGNN_ACT_NONE;
  bool vec = (p.C % 4 == 0) && (p.ldx % 4 == 0) && (p.x_type_stride % 4 == 0) && (p.ldo % 4 == 0) &&
             (p.out_type_stride % 4 == 0) && aligned16(p.X) && aligned16(p.out) && p.C <= 128 * 4;
  if (p.T) vec = vec && (p.ldt % 4 == 0) && (p.t_type_stride % 4 == 0) && aligned16(p.T);
  if (p.G) vec = vec && (p.ldg % 4 == 0) && (p.g_type_stride % 4 == 0) && (p.beta_off % 4 == 0) && aligned16(p.G);
  TFGNN_REQUIRE(!p.ties || (merged && p.reduce_max && vec),
                "the tie count is built for the merged max reduce with 16-byte rows of at most 512 columns");
  if (!vec) {
    const long long total = items * p.C;
    const int blocks = ceil_div(total, 256);
    if (merged) edge_reduce_scalar_kernel<true><<<blocks, 256, 0, st>>>(p);
    else edge_reduce_scalar_kernel<false><<<blocks, 256, 0, st>>>(p);
    TFGNN_LAUNCH_CHECK();
    return 0;
  }
  const int nv = (p.C + 127) / 128;
  static const bool lean = [] { const char* e = getenv("TFGNN_B200_GATHER_LEAN"); return !e || atoi(e) != 0; }();
  int blocks = ceil_div(items * 32, 256);
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
#define TFGNN_ER_LAUNCH(NV)                                                              \
  do {                                                                                   \
    if (merged && p.ties) edge_reduce_kernel<NV, true, false, 4, 1, true><<<blocks, 256, 0, st>>>(p); \
    else if (merged) edge_reduce_kernel<NV, true, false><<<blocks, 256, 0, st>>>(p);     \
    else if (plain && lean) edge_reduce_kernel<NV, false, true, 2, (NV == 1 ? 6 : 5)><<<blocks, 256, 0, st>>>(p); \
    else if (plain) edge_reduce_kernel<NV, false, true><<<blocks, 256, 0, st>>>(p);      \
    else edge_reduce_kernel<NV, false, false><<<blocks, 256, 0, st>>>(p);                \
  } while (0)
  switch (nv) {
    case 1: TFGNN_ER_LAUNCH(1); break;
    case 2: TFGNN_ER_LAUNCH(2); break;
    case 3: TFGNN_ER_LAUNCH(3); break;
    default: TFGNN_ER_LAUNCH(4); break;
  }
#undef TFGNN_ER_LAUNCH
  TFGNN_LAUNCH_CHECK();
  return 0;
}

int launch_edge_grad(const EdgeReduceParams& f, const float* z, const float* dz, const int* row_ptr_t, const int* tgt,
                     int Vs, float* out, cudaStream_t st) {
  TFGNN_REQUIRE(f.edge_act != TFGNN_ACT_NONE || f.reduce_max,
                "edge_grad differentiates the transform-then-aggregate reduce (max or activation before aggregation)");
  TFGNN_REQUIRE(!f.hidden_relu && !f.G && f.v_begin == 0 && (f.v_count == 0 || f.v_count == f.V),
                "edge_grad differentiates a whole-range reduce without hidden layer or FiLM");
  TFGNN_REQUIRE((z != nullptr) == (f.reduce_max != 0) && dz && out, "edge_grad: NULL pointer");
  bool vec = f.C % 4 == 0 && f.C <= 128 * 4 && f.ldx % 4 == 0 && f.x_type_stride % 4 == 0 && aligned16(f.X) &&
             aligned16(dz) && aligned16(out) && (!z || aligned16(z));
  if (f.T) vec = vec && f.ldt % 4 == 0 && f.t_type_stride % 4 == 0 && aligned16(f.T);
  TFGNN_REQUIRE(vec, "edge_grad needs 16-byte rows of at most 512 columns");
  const bool key_src = row_ptr_t != nullptr;
  const EdgeGradArgs a{f, z, dz, key_src ? row_ptr_t : f.row_ptr, key_src ? tgt : f.src, key_src ? Vs : f.V, out};
  const long long items = (long long)f.L * a.Vk;
  if (items == 0) return 0;
  long long blocks = (items * 32 + 255) / 256;
  if (blocks > 132 * 64) blocks = 132 * 64;
#define TFGNN_EG_LAUNCH(NV)                                                      \
  do {                                                                           \
    if (key_src) edge_grad_kernel<NV, true><<<(int)blocks, 256, 0, st>>>(a);     \
    else edge_grad_kernel<NV, false><<<(int)blocks, 256, 0, st>>>(a);            \
  } while (0)
  switch ((f.C + 127) / 128) {
    case 1: TFGNN_EG_LAUNCH(1); break;
    case 2: TFGNN_EG_LAUNCH(2); break;
    case 3: TFGNN_EG_LAUNCH(3); break;
    default: TFGNN_EG_LAUNCH(4); break;
  }
#undef TFGNN_EG_LAUNCH
  TFGNN_LAUNCH_CHECK();
  return 0;
}

int launch_target_term(const float* h, int ldh, const int* row_ptr, int V, int L, int D, int normalize,
                       float* out, int ldo, int col0, cudaStream_t st, int in_stride) {
  const long long total = (long long)V * L * D;
  if (total == 0) return 0;
  if (D % 4 == 0 && ldh % 4 == 0 && ldo % 4 == 0 && col0 % 4 == 0 && in_stride % 4 == 0 && aligned16(h) &&
      aligned16(out)) {
    int blocks = ceil_div((long long)V * 32, 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    target_term_vec_kernel<<<blocks, 256, 0, st>>>(h, ldh, row_ptr, V, L, D, normalize, out, ldo, col0, in_stride);
    TFGNN_LAUNCH_CHECK();
    return 0;
  }
  target_term_kernel<<<ceil_div(total, 256), 256, 0, st>>>(h, ldh, row_ptr, V, L, D, normalize, out, ldo, col0,
                                                            in_stride);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

int launch_edge_scatter_atomic(const tfgnn_batch* b, const float* X, int ldx, int C, int normalize,
                               float* out, int ldo, int type_stride, cudaStream_t st) {
  TFGNN_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && type_stride % 4 == 0 && aligned16(X) && aligned16(out),
                "atomic path needs 16-byte aligned rows (column counts divisible by 4)");
  for (int l = 0; l < b->L; ++l) {
    if (b->E[l] == 0) continue;
    int blocks = ceil_div(b->E[l] * 32, 256);
    if (blocks > 132 * 64) blocks = 132 * 64;
    edge_scatter_atomic_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const int2*>(b->adj[l]), b->E[l], l,
                                                        (int)b->V, X, ldx, C, b->row_ptr, normalize, out, ldo,
                                                        l * type_stride);
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace tfgnn
