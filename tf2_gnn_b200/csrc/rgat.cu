// RGAT aggregation (rgat.py:125-163): softmax over ALL incoming edges of a target (all edge types jointly),
// per head, then the attention-weighted sum of the projected source rows.
//
// Node-level part (variants.cu): P_l = h W_l for every node once, and the per-edge score is split by linearity
// of the einsum (rgat.py:115-121) into node-level halves s_src[u,l,k] + s_tgt[v,l,k].
//
// Edge-level part (this file), HBM-bound: per edge 4 B index + 4*K B of source scores + 4*H B of P row.  The forward and the
// backward's statistics share ONE target walk (rgat_warp_kernel):
//   * regular targets (in-degree <= kHubThreshold): one warp per target, lanes over float4 column groups, one pass over
//     the CSR segments with a running maximum ("online softmax"): when the maximum grows, the sums so far are rescaled by
//     exp(m_old - m_new), so every edge's score and P row are read once.
//   * hub targets (power-law graphs: up to 1e5+ incoming edges): the joint edge list is cut into chunks of kHubChunk edges,
//     one warp per chunk; each chunk writes its partial and the partials are combined in chunk order
//     (rgat_hub_combine_kernel).  Without this a single warp would walk a hub serially for ~50 ms.
// No float atomics: every result is bitwise reproducible.
//
// Backward (tfgnn_b200_rgat_bwd, backward.cu).  For an edge e = (u -> v) of type l and head k: x_e = s_src[u,l,k] +
// s_tgt[v,l,k], sigma_e = leaky(x_e), alpha_e = exp(sigma_e - m[v,k]) / den[v,k], and with dZ = dOut * act':
//   da_e = dZ[v]_k . P_l[u]_k,   g[v,k] = sum_e alpha_e da_e,   dx_e = alpha_e (da_e - g[v,k]) leaky'(x_e)
//   ds_tgt[v,l,k] = sum over the edges of type l into v of dx_e                      (target walk, statistics mode)
//   ds_src[u,l,k] = sum over the edges of type l leaving u of dx_e,
//   dP_l[u]_k = sum over those edges of alpha_e dZ[v]_k + ds_src[u,l,k] a_l[k,:d] + ds_tgt[u,l,k] a_l[k,d:]   (source pass)
// In statistics mode the walk keeps den = sum w_e, G = sum w_e da_e and, for the type being walked, A1 = sum w_e leaky'(x_e)
// da_e and A2 = sum w_e leaky'(x_e), all rescaled by exp(m_old - m_new) when the maximum grows.  At the end of each type A1,
// A2 and the maximum they refer to are flushed to memory; after the walk they are brought to the final maximum: g = G / den,
// ds_tgt = (A1 - g A2) / den.  A hub chunk's partial is (m_c, den_c, G_c, A1_c, A2_c).  A head's dot product (d columns =
// d/4 float4 groups) is summed inside the warp by rgat_head_sum.
#include "layers.cuh"

namespace tfgnn {

constexpr int kHubThreshold = 2048;
constexpr int kHubChunk = 1024;
constexpr int kRgatRowChunk = 8192;   // rows per partial of the attention gradient

__device__ __forceinline__ float rgat_leaky(float x) { return x > 0.f ? x : kLeakyReluAlpha * x; }

struct RgatWalkParams {
  const float* P;       // [Vs, L*H]
  const float* s_src;   // [Vs, L*K]
  const float* s_tgt;   // [Vs, L*K]
  const int* row_ptr;
  const int* src;
  long long V, tgt_off;
  int L, K, d, H;
  int act;              // output mode: activation of out
  float* out;           // output mode: [V, H]
  const float* dz;      // [V, H]; NULL: output mode
  float* stat;          // [V, 3K]: m, den, g per head
  float* a1;            // [V, L*K]: flushed A1 of regular targets, then ds_tgt
  float* a2;            // [V, L*K]: flushed A2
  float* ml;            // [V, L*K]: the maximum A1, A2 refer to
  const int2* items;    // hub chunks (target, chunk), the chunks of a hub consecutive
  const int* item_count;
  float* hstat;         // [items, 3K]: m_c, den_c, G_c
  float* ha1;           // [items, L*K] (output mode: the un-normalised row acc_c [items, H])
  float* ha2;
  float* hml;
};

// v[j], this lane's partial for column group q = lane + 32 j, becomes the sum over the g = d/4 groups of q's head, with the
// same bits in every lane of the head.  Power-of-two g: a butterfly inside aligned groups of g lanes (commutative at every
// level, so every lane gets the same bits), then over the j of a head when it spans several; otherwise through the warp's
// row `red` (32 NV floats) in column order.
template <int NV>
__device__ __forceinline__ void rgat_head_sum(float (&v)[NV], int lane, int g, float* red) {
  if ((g & (g - 1)) == 0) {
    const int w = g < 32 ? g : 32;
#pragma unroll
    for (int j = 0; j < NV; ++j)
      for (int o = w >> 1; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
    if (g > 32) {
      const int span = g >> 5;
      float t[NV];
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        t[j] = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i)
          if (i / span == j / span) t[j] += v[i];
      }
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = t[j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < NV; ++j) red[32 * j + lane] = v[j];
    __syncwarp();
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int h0 = (lane + 32 * j) / g * g;
      float s = 0.f;
      for (int i = h0; i < h0 + g && i < 32 * NV; ++i) s += red[i];
      v[j] = s;
    }
    __syncwarp();
  }
}

__device__ __forceinline__ float dot4(float4 a, float4 b) {
  return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}

// Hub discovery: one thread per target; a hub gets ceil(deg / kHubChunk) consecutive work items.
__global__ void rgat_hub_scan_kernel(const int* __restrict__ row_ptr, long long V, int L, int2* __restrict__ items,
                                     int* __restrict__ item_count) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    int deg = 0;
    for (int l = 0; l < L; ++l) deg += row_ptr[(long long)l * V + v + 1] - row_ptr[(long long)l * V + v];
    if (deg <= kHubThreshold) continue;
    const int nchunks = (deg + kHubChunk - 1) / kHubChunk;
    const int base = atomicAdd(item_count, nchunks);   // integer work-list slot; the values never depend on it
    for (int c = 0; c < nchunks; ++c) items[base + c] = make_int2((int)v, c);
  }
}

// The target walk: one warp per (work item, column block of 32 NV float4 groups, blockIdx.y), where a work item is a
// regular target (w < V) or a hub chunk (w >= V); NV groups per lane.
//   output mode (!STATS, the forward): act(o) of regular rows into out, the partial (m_c, den_c, acc_c) of hub chunks; the
//     score and P-row loads of 4 edges are issued before they are used.
//   statistics mode (STATS, the backward; one column block, so a head's dot product stays in the warp): stat and ds_tgt.
// Both modes apply the same operations per edge, so the backward's statistics refer to the forward's bits.
template <int NV, bool STATS>
__global__ void __launch_bounds__(256) rgat_warp_kernel(const RgatWalkParams p) {
  constexpr int EB = STATS ? 1 : 4;   // edges per batch of loads
  __shared__ float red_all[8][32 * NV];
  const int lane = threadIdx.x & 31;
  float* red = red_all[threadIdx.x >> 5];
  const long long LK = (long long)p.L * p.K, LH = (long long)p.L * p.H;
  const int C4 = p.H >> 2, g = p.d >> 2, K3 = 3 * p.K;
  const long long n_work = p.V + *p.item_count;
  int q[NV], k[NV];
  bool ok[NV], lead[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    q[j] = lane + 32 * (blockIdx.y * NV + j);
    ok[j] = q[j] < C4;
    k[j] = ok[j] ? q[j] / g : 0;
    lead[j] = ok[j] && q[j] % g == 0;   // the head's first lane writes its per-head values
  }
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_work;
       w += ((long long)gridDim.x * blockDim.x) >> 5) {
    const bool hub = w >= p.V;
    long long v;
    int r_lo = 0, r_hi = 0x7fffffff;   // rank range in the joint edge list of v, then in the rest of it
    if (!hub) {
      v = w;
      int deg = 0;
      for (int l = 0; l < p.L; ++l) deg += __ldg(p.row_ptr + (long long)l * p.V + v + 1) - __ldg(p.row_ptr + (long long)l * p.V + v);
      if (deg > kHubThreshold) continue;   // walked by its chunks
    } else {
      const int2 item = p.items[w - p.V];
      v = item.x;
      r_lo = item.y * kHubChunk;
      r_hi = r_lo + kHubChunk;
    }
    const long long row = hub ? w - p.V : v;
    float* fa1 = (hub ? p.ha1 : p.a1) + row * LK;
    float* fa2 = (hub ? p.ha2 : p.a2) + row * LK;
    float* fml = (hub ? p.hml : p.ml) + row * LK;
    float4 z[NV], acc[NV];
    float m[NV], den[NV], G[NV], A1[NV], A2[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      z[j] = (STATS && ok[j]) ? ldg_f4(p.dz + v * p.H + 4 * q[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      m[j] = kLowestFloat;
      den[j] = G[j] = 0.f;
    }
    for (int l = 0; l < p.L; ++l) {
      const long long seg = (long long)l * p.V + v;
      const int beg = __ldg(p.row_ptr + seg), end = __ldg(p.row_ptr + seg + 1);
      const int e_lo = beg + max(r_lo, 0), e_hi = beg + min(r_hi, end - beg);
      r_lo -= end - beg;
      r_hi -= end - beg;
      float st[NV];
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        A1[j] = A2[j] = 0.f;
        st[j] = (ok[j] && e_lo < e_hi) ? __ldg(p.s_tgt + (v + p.tgt_off) * LK + l * p.K + k[j]) : 0.f;
      }
      for (int base = e_lo; base < e_hi; base += 32) {
        const int n = min(32, e_hi - base);
        const int my_src = lane < n ? __ldg(p.src + base + lane) : 0;
        for (int e0 = 0; e0 < n; e0 += EB) {
          float sc[EB][NV];
          float4 x[EB][NV];
#pragma unroll
          for (int i = 0; i < EB; ++i) {
            const long long u = __shfl_sync(0xffffffffu, my_src, (e0 + i) & 31);
#pragma unroll
            for (int j = 0; j < NV; ++j) {
              const bool in = ok[j] && e0 + i < n;
              sc[i][j] = in ? __ldg(p.s_src + u * LK + l * p.K + k[j]) : 0.f;
              x[i][j] = in ? ldg_f4(p.P + u * LH + (long long)l * p.H + 4 * q[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
#pragma unroll
          for (int i = 0; i < EB; ++i) {
            if (e0 + i >= n) break;
            float da[NV];
            if (STATS) {
#pragma unroll
              for (int j = 0; j < NV; ++j) da[j] = dot4(z[j], x[i][j]);
              rgat_head_sum<NV>(da, lane, g, red);
            }
#pragma unroll
            for (int j = 0; j < NV; ++j) {
              const float xs = sc[i][j] + st[j];
              const float score = rgat_leaky(xs);
              const float lp = xs > 0.f ? 1.f : kLeakyReluAlpha;
              const float4 xe = x[i][j];
              if (score > m[j]) {   // this edge weighs exp(0) = 1, the sums so far are rescaled (the first edge: by 0)
                const float r = expf(m[j] - score);
                m[j] = score;
                den[j] = fmaf(den[j], r, 1.0f);
                if (STATS) {
                  G[j] = fmaf(G[j], r, da[j]);
                  A1[j] = fmaf(A1[j], r, lp * da[j]);
                  A2[j] = fmaf(A2[j], r, lp);
                } else {
                  acc[j].x = fmaf(acc[j].x, r, xe.x); acc[j].y = fmaf(acc[j].y, r, xe.y);
                  acc[j].z = fmaf(acc[j].z, r, xe.z); acc[j].w = fmaf(acc[j].w, r, xe.w);
                }
              } else {
                const float wt = expf(score - m[j]);
                den[j] += wt;
                if (STATS) {
                  G[j] = fmaf(wt, da[j], G[j]);
                  A1[j] = fmaf(wt, lp * da[j], A1[j]);
                  A2[j] = fmaf(wt, lp, A2[j]);
                } else {
                  acc[j].x = fmaf(wt, xe.x, acc[j].x); acc[j].y = fmaf(wt, xe.y, acc[j].y);
                  acc[j].z = fmaf(wt, xe.z, acc[j].z); acc[j].w = fmaf(wt, xe.w, acc[j].w);
                }
              }
            }
          }
        }
      }
      if (STATS) {
#pragma unroll
        for (int j = 0; j < NV; ++j)
          if (lead[j]) {
            const int i = l * p.K + k[j];
            fa1[i] = A1[j];
            fa2[i] = A2[j];
            fml[i] = m[j];
          }
      }
    }
    if (!STATS) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        if (!ok[j]) continue;
        if (!hub) {
          const float inv = den[j] > 0.f ? 1.0f / den[j] : 0.f;
          float o[4] = {acc[j].x * inv, acc[j].y * inv, acc[j].z * inv, acc[j].w * inv};
          apply_act_vec<4>(o, p.act);
          *reinterpret_cast<float4*>(p.out + v * p.H + 4 * q[j]) = make_float4(o[0], o[1], o[2], o[3]);
        } else {
          *reinterpret_cast<float4*>(p.ha1 + row * p.H + 4 * q[j]) = acc[j];
          if (lead[j]) {   // every column block holding the head computes the same m_c, den_c bits
            p.hstat[row * K3 + k[j]] = m[j];
            p.hstat[row * K3 + p.K + k[j]] = den[j];
          }
        }
      }
      continue;
    }
    // bring the flushed per-type sums to the final maximum (this thread reads back what it wrote)
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      if (!lead[j]) continue;
      const float gk = den[j] > 0.f ? G[j] / den[j] : 0.f;
      const float inv = den[j] > 0.f ? 1.0f / den[j] : 0.f;
      for (int l = 0; l < p.L; ++l) {
        const int i = l * p.K + k[j];
        const float s = expf(fml[i] - m[j]);
        const float a1 = fa1[i] * s, a2 = fa2[i] * s;
        if (hub) {
          fa1[i] = a1;
          fa2[i] = a2;
        } else {
          fa1[i] = (a1 - gk * a2) * inv;
        }
      }
      float* sr = (hub ? p.hstat : p.stat) + row * K3;
      sr[k[j]] = m[j];
      sr[p.K + k[j]] = den[j];
      sr[2 * p.K + k[j]] = hub ? G[j] : gk;
    }
  }
}

// The chunks of every hub combined in chunk order: act(o) of the hub's row (output mode) or its stat and ds_tgt.
template <bool STATS>
__global__ void rgat_hub_combine_kernel(const RgatWalkParams p) {
  const int count = *p.item_count;
  const long long LK = (long long)p.L * p.K;
  const int K3 = 3 * p.K;
  for (int it = blockIdx.x; it < count; it += gridDim.x) {
    const int2 item = p.items[it];
    if (item.y != 0) continue;   // once per hub; its chunks are items it, it + 1, ..
    const long long v = item.x;
    int deg = 0;
    for (int l = 0; l < p.L; ++l) deg += p.row_ptr[(long long)l * p.V + v + 1] - p.row_ptr[(long long)l * p.V + v];
    const int nch = (deg + kHubChunk - 1) / kHubChunk;
    if (!STATS) {
      for (int c = threadIdx.x; c < p.H; c += blockDim.x) {
        const int k = c / p.d;
        float m = kLowestFloat;
        for (int i = 0; i < nch; ++i) m = fmaxf(m, p.hstat[(it + i) * K3 + k]);
        float den = 0.f, acc = 0.f;
        for (int i = 0; i < nch; ++i) {
          const float s = expf(p.hstat[(it + i) * K3 + k] - m);
          den = fmaf(p.hstat[(it + i) * K3 + p.K + k], s, den);
          acc = fmaf(p.ha1[(long long)(it + i) * p.H + c], s, acc);
        }
        float o[1] = {den > 0.f ? acc * (1.0f / den) : 0.f};
        apply_act_vec<1>(o, p.act);
        p.out[v * p.H + c] = o[0];
      }
      continue;
    }
    for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
      float m = kLowestFloat;
      for (int i = 0; i < nch; ++i) m = fmaxf(m, p.hstat[(it + i) * K3 + k]);
      float den = 0.f, G = 0.f;
      for (int i = 0; i < nch; ++i) {
        const float s = expf(p.hstat[(it + i) * K3 + k] - m);
        den = fmaf(p.hstat[(it + i) * K3 + p.K + k], s, den);
        G = fmaf(p.hstat[(it + i) * K3 + 2 * p.K + k], s, G);
      }
      const float gk = den > 0.f ? G / den : 0.f;
      const float inv = den > 0.f ? 1.0f / den : 0.f;
      p.stat[v * K3 + k] = m;
      p.stat[v * K3 + p.K + k] = den;
      p.stat[v * K3 + 2 * p.K + k] = gk;
      for (int l = 0; l < p.L; ++l) {
        float a1 = 0.f, a2 = 0.f;
        for (int i = 0; i < nch; ++i) {
          const float s = expf(p.hstat[(it + i) * K3 + k] - m);
          a1 = fmaf(p.ha1[(it + i) * LK + l * p.K + k], s, a1);
          a2 = fmaf(p.ha2[(it + i) * LK + l * p.K + k], s, a2);
        }
        p.a1[v * LK + l * p.K + k] = (a1 - gk * a2) * inv;
      }
    }
  }
}

struct RgatSrcParams {
  const float* P;
  const float* s_src;
  const float* s_tgt;
  const int* row_ptr_t;   // source-keyed CSR: segment (l, u) = l*Vs + u, values = local target ids
  const int* tgt;
  long long Vs, V, tgt_off;
  int L, K, d, H;
  const float* dz;        // [V, H]
  const float* stat;      // [V, 3K]
  const float* ds_tgt;    // [V, L*K]
  PtrTable att;           // a_l [K, 2d]
  float* dP;              // [Vs, L*H]
  float* ds_src;          // [Vs, L*K]
};

// Source pass: one warp per (type, source) segment of the source-keyed CSR, in canonical order; P_l[u] stays in registers.
template <int NV>
__global__ void __launch_bounds__(256) rgat_bwd_source_kernel(const RgatSrcParams p) {
  __shared__ float red_all[8][32 * NV];
  const int lane = threadIdx.x & 31;
  float* red = red_all[threadIdx.x >> 5];
  const long long LK = (long long)p.L * p.K, LH = (long long)p.L * p.H;
  const int C4 = p.H >> 2, g = p.d >> 2, K3 = 3 * p.K;
  int q[NV], k[NV];
  bool ok[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    q[j] = lane + 32 * j;
    ok[j] = q[j] < C4;
    k[j] = ok[j] ? q[j] / g : 0;
  }
  const long long items = (long long)p.L * p.Vs;
  for (long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < items;
       item += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int l = (int)(item / p.Vs);
    const long long u = item - (long long)l * p.Vs;
    const int beg = __ldg(p.row_ptr_t + item), end = __ldg(p.row_ptr_t + item + 1);
    const float* prow = p.P + u * LH + (long long)l * p.H;
    float4 key[NV], acc[NV];
    float ss[NV], dsrc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      key[j] = ok[j] ? ldg_f4(prow + 4 * q[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
      ss[j] = ok[j] ? __ldg(p.s_src + u * LK + l * p.K + k[j]) : 0.f;
      acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      dsrc[j] = 0.f;
    }
    for (int base = beg; base < end; base += 32) {
      const int n = min(32, end - base);
      const int my_tgt = lane < n ? __ldg(p.tgt + base + lane) : 0;
      for (int e = 0; e < n; ++e) {
        const long long v = __shfl_sync(0xffffffffu, my_tgt, e);
        float4 zr[NV];
        float da[NV], mx[NV], dn[NV], gk[NV], st[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          zr[j] = ok[j] ? ldg_f4(p.dz + v * p.H + 4 * q[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
          st[j] = ok[j] ? __ldg(p.s_tgt + (v + p.tgt_off) * LK + l * p.K + k[j]) : 0.f;
          mx[j] = ok[j] ? __ldg(p.stat + v * K3 + k[j]) : 0.f;
          dn[j] = ok[j] ? __ldg(p.stat + v * K3 + p.K + k[j]) : 1.f;
          gk[j] = ok[j] ? __ldg(p.stat + v * K3 + 2 * p.K + k[j]) : 0.f;
          da[j] = dot4(zr[j], key[j]);
        }
        rgat_head_sum<NV>(da, lane, g, red);
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const float xs = ss[j] + st[j];
          const float lp = xs > 0.f ? 1.f : kLeakyReluAlpha;
          const float alpha = expf(rgat_leaky(xs) - mx[j]) / dn[j];
          dsrc[j] = fmaf(alpha * (da[j] - gk[j]), lp, dsrc[j]);
          acc[j].x = fmaf(alpha, zr[j].x, acc[j].x); acc[j].y = fmaf(alpha, zr[j].y, acc[j].y);
          acc[j].z = fmaf(alpha, zr[j].z, acc[j].z); acc[j].w = fmaf(alpha, zr[j].w, acc[j].w);
        }
      }
    }
    // dP_l[u] = acc + ds_src a_l[k,:d] + ds_tgt a_l[k,d:]  (the target term on the rows this batch owns)
    const long long own = u - p.tgt_off;
    const bool owned = own >= 0 && own < p.V;
    const float* a = reinterpret_cast<const float*>(p.att.p[l]);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      if (!ok[j]) continue;
      const float* as = a + (long long)k[j] * 2 * p.d + (4 * q[j] - k[j] * p.d);
      const float* at = as + p.d;
      const float dt = owned ? __ldg(p.ds_tgt + own * LK + l * p.K + k[j]) : 0.f;
      const float4 o = make_float4(fmaf(dt, __ldg(at), fmaf(dsrc[j], __ldg(as), acc[j].x)),
                                   fmaf(dt, __ldg(at + 1), fmaf(dsrc[j], __ldg(as + 1), acc[j].y)),
                                   fmaf(dt, __ldg(at + 2), fmaf(dsrc[j], __ldg(as + 2), acc[j].z)),
                                   fmaf(dt, __ldg(at + 3), fmaf(dsrc[j], __ldg(as + 3), acc[j].w)));
      *reinterpret_cast<float4*>(p.dP + u * LH + (long long)l * p.H + 4 * q[j]) = o;
      if (q[j] % g == 0) p.ds_src[u * LK + l * p.K + k[j]] = dsrc[j];
    }
  }
}

// part[c][col] = sum over the rows r of chunk c (kRgatRowChunk rows) of ds[r, l, k] P[r, col], col = l*H + k*d + i
__global__ void rgat_att_grad_partial_kernel(const float* __restrict__ ds, const float* __restrict__ P, long long rows, int L,
                                             int K, int d, float* __restrict__ part) {
  const int H = K * d, LH = L * H;
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= LH) return;
  const int l = col / H, k = (col - l * H) / d;
  const long long LK = (long long)L * K;
  const long long r0 = (long long)blockIdx.y * kRgatRowChunk;
  const long long r1 = r0 + kRgatRowChunk < rows ? r0 + kRgatRowChunk : rows;
  float s = 0.f;
  for (long long r = r0; r < r1; ++r) s = fmaf(ds[r * LK + l * K + k], P[r * LH + col], s);
  part[(long long)blockIdx.y * LH + col] = s;
}

// grad_att[l][k, half*d + i] = sum over the chunks, in chunk order
__global__ void rgat_att_grad_reduce_kernel(const float* __restrict__ part, int chunks, int L, int K, int d, PtrTable grad_att,
                                            int half) {
  const int H = K * d, LH = L * H;
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= LH) return;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += part[(long long)c * LH + col];
  const int l = col / H, k = (col - l * H) / d, i = col - l * H - k * d;
  reinterpret_cast<float*>(const_cast<void*>(grad_att.p[l]))[(long long)k * 2 * d + half * d + i] = s;
}

static int rgat_bwd_blocks(long long warps) {
  const long long g = (warps * 32 + 255) / 256;
  return g < 1 ? 1 : (g > 132 * 64 ? 132 * 64 : (int)g);
}

// One target walk over the batch (rgat_warp_kernel) and the chunk-order combine of its hub partials; p.dz NULL: output mode.
static int rgat_target_walk(tfgnn_batch* b, RgatWalkParams& p, cudaStream_t st) {
  const bool stats = p.dz != nullptr;
  p.row_ptr = b->row_ptr; p.src = b->src_sorted;
  p.V = b->V; p.tgt_off = b->tgt_off; p.L = b->L; p.H = p.K * p.d;
  const long long LK = (long long)p.L * p.K;
  // a hub has more than kHubThreshold edges and at most deg / kHubChunk + 1 chunks
  const long long max_items = b->M_in / kHubChunk + b->M_in / kHubThreshold + 2;
  PoolBuffer items{st}, hub{st}, flush{st};
  int rc = items.alloc((size_t)max_items * sizeof(int2) + 16);
  if (rc) return rc;
  // per hub chunk: A1_c, A2_c and their maximum (output mode: the [H] row acc_c, stored as float4: so the rows come first),
  // then m_c, den_c, G_c
  const size_t hub_row = stats ? (size_t)3 * LK : (size_t)p.H;
  rc = hub.alloc((size_t)max_items * (hub_row + 3 * p.K) * sizeof(float));
  if (rc) return rc;
  p.ha1 = hub.f();
  p.hstat = hub.f() + (size_t)max_items * hub_row;
  if (stats) {
    p.ha2 = p.ha1 + (size_t)max_items * LK;
    p.hml = p.ha2 + (size_t)max_items * LK;
    rc = flush.alloc((size_t)2 * p.V * LK * sizeof(float));
    if (rc) return rc;
    p.a2 = flush.f();
    p.ml = flush.f() + (size_t)p.V * LK;
  }
  p.item_count = (int*)items.p;
  p.items = reinterpret_cast<const int2*>(reinterpret_cast<char*>(items.p) + 16);
  TFGNN_CUDA(cudaMemsetAsync(items.p, 0, sizeof(int), st));
  rgat_hub_scan_kernel<<<grid_for(p.V), 256, 0, st>>>(p.row_ptr, p.V, p.L, const_cast<int2*>(p.items),
                                                     const_cast<int*>(p.item_count));
  TFGNN_LAUNCH_CHECK();
  if (stats) {
    const int blocks = rgat_bwd_blocks(p.V + max_items);
    switch ((p.H + 127) / 128) {
      case 1: rgat_warp_kernel<1, true><<<blocks, 256, 0, st>>>(p); break;
      case 2: rgat_warp_kernel<2, true><<<blocks, 256, 0, st>>>(p); break;
      case 3: rgat_warp_kernel<3, true><<<blocks, 256, 0, st>>>(p); break;
      case 4: rgat_warp_kernel<4, true><<<blocks, 256, 0, st>>>(p); break;
      default: return unsupported("rgat_bwd: hidden_dim above 512 is not built");
    }
    TFGNN_LAUNCH_CHECK();
    rgat_hub_combine_kernel<true><<<132, 128, 0, st>>>(p);
  } else {
    // one warp per (work item, 128-column block)
    const dim3 grid((unsigned)ceil_div((p.V + max_items) * 32, 256), (unsigned)ceil_div(p.H, 128));
    rgat_warp_kernel<1, false><<<grid, 256, 0, st>>>(p);
    TFGNN_LAUNCH_CHECK();
    rgat_hub_combine_kernel<false><<<132, 128, 0, st>>>(p);
  }
  TFGNN_LAUNCH_CHECK();
  return 0;
}

int launch_rgat_aggregate(tfgnn_batch* b, const float* P, const float* s_src, const float* s_tgt, int K, int d,
                          int activation, float* out, cudaStream_t st) {
  RgatWalkParams p{};
  p.P = P; p.s_src = s_src; p.s_tgt = s_tgt; p.K = K; p.d = d; p.act = activation; p.out = out;
  return rgat_target_walk(b, p, st);
}

int launch_rgat_target_pass(tfgnn_batch* b, const float* P, const float* s_src, const float* s_tgt, int K, int d,
                            const float* dz, float* stat, float* ds_tgt, cudaStream_t st) {
  TFGNN_REQUIRE(dz && stat && ds_tgt, "rgat target pass: NULL pointer");
  RgatWalkParams p{};
  p.P = P; p.s_src = s_src; p.s_tgt = s_tgt; p.K = K; p.d = d; p.dz = dz; p.stat = stat; p.a1 = ds_tgt;
  return rgat_target_walk(b, p, st);
}

int launch_rgat_source_pass(const tfgnn_batch* b, const tfgnn_batch* bt, const float* P, const float* s_src,
                            const float* s_tgt, const PtrTable& att, int K, int d, const float* dz, const float* stat,
                            const float* ds_tgt, float* dP, float* ds_src, cudaStream_t st) {
  RgatSrcParams p{};
  p.P = P; p.s_src = s_src; p.s_tgt = s_tgt; p.row_ptr_t = bt->row_ptr; p.tgt = bt->src_sorted;
  p.Vs = b->V_src; p.V = b->V; p.tgt_off = b->tgt_off; p.L = b->L; p.K = K; p.d = d; p.H = K * d;
  p.dz = dz; p.stat = stat; p.ds_tgt = ds_tgt; p.att = att; p.dP = dP; p.ds_src = ds_src;
  const int blocks = rgat_bwd_blocks((long long)p.L * p.Vs);
  switch ((p.H + 127) / 128) {
    case 1: rgat_bwd_source_kernel<1><<<blocks, 256, 0, st>>>(p); break;
    case 2: rgat_bwd_source_kernel<2><<<blocks, 256, 0, st>>>(p); break;
    case 3: rgat_bwd_source_kernel<3><<<blocks, 256, 0, st>>>(p); break;
    case 4: rgat_bwd_source_kernel<4><<<blocks, 256, 0, st>>>(p); break;
    default: return unsupported("rgat_bwd: hidden_dim above 512 is not built");
  }
  TFGNN_LAUNCH_CHECK();
  return 0;
}

int launch_rgat_attention_grad(const float* ds, const float* P, long long rows, int L, int K, int d, const PtrTable& grad_att,
                               int half, cudaStream_t st) {
  const int LH = L * K * d;
  const int chunks = rows > 0 ? ceil_div(rows, kRgatRowChunk) : 1;
  PoolBuffer part{st};
  int rc = part.alloc((size_t)chunks * LH * sizeof(float));
  if (rc) return rc;
  rgat_att_grad_partial_kernel<<<dim3(ceil_div(LH, 128), chunks), 128, 0, st>>>(ds, P, rows, L, K, d, part.f());
  TFGNN_LAUNCH_CHECK();
  rgat_att_grad_reduce_kernel<<<ceil_div(LH, 128), 128, 0, st>>>(part.f(), chunks, L, K, d, grad_att, half);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn
