// The fused RGCN-style layer: ONE persistent kernel does gather(h[src]) -> segment-sum -> 1/(c+eps)
// -> 3xTF32 wgmma contraction with [W_0;..;W_{L-1}] -> row-norm / activation -> out.
//
//   out[v] = act( rn(v) * sum_l ( 1/(c_{v,l}+eps) * sum_{(u,v) in A_l} h_u ) W_l )       (rgcn.py:13-48)
//
// One CTA per SM owns 128-target tiles.  Inside the CTA, 8 GATHER warps produce, per edge type l, the normalised row sums
// A_l[128, D] (full 4*D-byte row reads from HBM through a rolling cp.async ring in shared memory, register accumulation, no
// atomics) into a small per-CTA ring in global memory that is meant to stay L2-resident (the fp32-accurate operand does not
// fit the 227 KB of shared memory next to the pipeline).  The TMA producer pulls each slot back in 128 B K-slices next to the
// pre-split weight tile; two consumer warpgroups (64 rows each) cut their rows of A into tf32 hi / lo in place and issue the
// wgmma of the K block into main + correction accumulators in registers, then run the epilogue straight from those
// registers.  The gather of the next slots overlaps the MMAs of slot i, and the [V, L*D] intermediate never touches HBM.
// The accumulators of a 64 x BN half tile take BN registers per thread, and with 17 warps a thread has 96 (five warps share
// an SM quarter's register file), so a tile is at most 64 columns wide: wider layers take several N passes over the same
// gathered ring slots (the ring then holds all L types of the tile).  Layers with 64 < H <= 256 (H % 32 == 0) outside
// split-tile mode take fused_rgcn_rows_kernel instead: one pass over all H columns, a CTA pair splitting each 128-row tile
// by columns (see there).
//
// Warp roles (544 threads):
//   0-7: two consumer warpgroups (split, MMA, epilogue) | 8: TMA | 9-16: gather.
// The gather warps hold no row data in registers while it is in flight: each keeps a rolling ring of cp.async
// copies into its own shared-memory slots (see GatherIssue), so DRAM requests in flight are bounded by the
// shared memory left over by the GEMM pipeline, not by registers.
#include <cuda.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "gemm.cuh"
#include "wgmma_tile.cuh"

namespace tfgnn {

constexpr int kFuBM = 128;
constexpr int kFuBK = 32;                       // floats per K block = one 128 B swizzle row
constexpr int kFuATileBytes = kFuBM * kFuBK * 4;
constexpr int kFuGatherWarps = 8;
constexpr int kFuFirstGatherWarp = 9;
constexpr int kFuThreads = 32 * (kFuFirstGatherWarp + kFuGatherWarps);
constexpr int kFuMaxSlots = 8;                  // ring slots per CTA: 4, or L+1 when the N dimension needs several passes
constexpr int kFuMaxBN = 64;                   // accumulators of a 64 x BN half tile: BN of the 96 registers
constexpr int kFuSmemLimit = 227 * 1024;
constexpr int kFuMaxQ = 8;                      // bulk row copies in flight per gather warp (upper bound)

struct FusedParams {
  // graph
  const float* h;
  int ldh;
  const int* row_ptr;
  const int* src;
  int V, L, D;
  int normalize;
  long long M;          // entries of src (bound for the 32-wide index block loads)
  int discard_ring;     // discard.global.L2 on consumed ring slots
  int gather_q;         // bulk row copies each gather warp keeps in flight (= its shared-memory row slots)
  int corr_bf16;        // 1: corrections as one bf16-pair MMA (sm90_ptx.cuh), 0: two tf32 MMAs
  int debug_skip;       // timing experiments only (results invalid), bit mask: 1 = no edge gathers, 2 = one K block per slot, 16 = no ring stores
  int split;            // split-tile mode: the two CTAs of a cluster share each tile (see fused_rgcn_kernel)
  // ring
  float* ring;  // [grid * num_slots * 128, D]
  int num_slots;
  // GEMM
  int N, cta_n, block_n, n_tiles;   // n_tiles: N passes of block_n columns over this CTA's cta_n columns
  long long m_tiles;
  int kb_per_type, num_stages;
  float* C;
  int ldc;
  // fused all-gather (tfgnn_b200_rgcn_fwd_allgather): peer copies of the output table, NVLink-mapped; same row indexing as C
  float* C_peer[TFGNN_MAX_PEERS];
  int n_peer;
  float* C_mc;   // multicast mapping of all replicas (NVSwitch replicates one multimem.st), or null
  uint32_t sleep_crit, sleep_long;   // nanosleep between barrier probes (0 = spin): K-loop waits / once-per-tile waits
  GemmEpilogue epi;
};

__device__ __forceinline__ float fu_row_norm(const GemmEpilogue& e, long long row) {
  if (e.row_norm == 0) return 1.0f;
  int cnt = 0;
  for (int l = 0; l < e.L; ++l) {
    const long long s = (long long)l * e.V + e.row0 + row;
    cnt += __ldg(e.row_ptr + s + 1) - __ldg(e.row_ptr + s);
  }
  const float c = (float)max(cnt, 1);
  return e.row_norm == 1 ? c : sqrtf(c);
}

// ---- gather warps: rolling cp.async ring ---------------------------------------------------------------------
// Each gather warp owns 8 consecutive targets of every tile and walks their CSR segments, one edge type after
// the other ("calls": (tile, type) -> one contiguous edge range).  Source rows do not wait in registers: the warp
// keeps Q rows in flight AT ALL TIMES as cp.async (LDGSTS) copies into its own Q shared-memory row slots - every
// lane copies and later reads back only its own 16-byte columns, one commit group per row, so
// `cp.async.wait_group Q-1` means "the oldest row has landed" and no mbarrier or warp barrier is needed.  When a
// row has been added to the register accumulator its slot is refilled at once with the row Q edges ahead, across
// segment, call and tile boundaries: the issue cursor and the consume cursor walk the same edge sequence
// independently, so the pipeline never drains.
// Summation order inside a segment is ascending CSR order, as in the unfused path.
struct GatherIssue {
  const int* row_ptr;
  const int* src;
  const float* h;        // + 4 * lane: this lane's first 16-byte column
  long long M;
  int V, L, ldh, skip, C4;
  int lane, gw, Q, ncalls;
  long long unit0, unit_step;
  int ctas, rank;
  int tile_rows;         // rows per tile (128, or 64 in the row tiling)
  int rpw, row_off;      // rows of the tile owned by this warp, first row of this CTA's share of the tile
  int w_row0;            // first row of this warp inside that share
  uint32_t buf_s;       // shared-window address of this warp's slot 0, + 16 * lane
  uint32_t row_bytes;
  int ic;                // call being issued
  int i_pos, i_end, in_blk, i_blk;
  int rpA, rpB, rpC;     // row_ptr[v0 + lane] of calls ic, ic+1, ic+2 (prefetched: the loads are two calls old when used)
  int ids, ids_next, ids0B;
  uint32_t ibuf;         // slot the next row goes to
  int islot;

  __device__ __forceinline__ void call_rows(int n, int& l, int& v0, int& nr) const {
    const int u = n / L;
    l = n - u * L;
    const long long tile = (unit0 + (long long)u * unit_step) * ctas + rank;
    v0 = (int)(tile * tile_rows) + row_off + w_row0;
    nr = V - v0;
    nr = nr < 0 ? 0 : (nr > rpw ? rpw : nr);
  }
  __device__ __forceinline__ int rp_of(int n) const {   // row_ptr of the call's rows, lane r -> first edge of row r
    if (n >= ncalls) return 0;
    int l, v0, nr;
    call_rows(n, l, v0, nr);
    if (nr == 0) return 0;
    const int* base = row_ptr + (long long)l * V + v0;
    return __ldg(base + (skip ? 0 : (lane <= nr ? lane : nr)));
  }
  __device__ __forceinline__ int nrows_of(int n) const {
    int l, v0, nr;
    call_rows(n, l, v0, nr);
    return nr;
  }
  __device__ __forceinline__ int load_ids(int first) const {
    const long long i = (long long)first + lane;
    return i < M ? __ldg(src + i) : 0;
  }
  __device__ __forceinline__ void next_call() {
    ++ic;
    rpA = rpB;
    rpB = rpC;
    rpC = rp_of(ic + 2);
    i_pos = __shfl_sync(0xffffffffu, rpA, 0);
    i_end = __shfl_sync(0xffffffffu, rpA, nrows_of(ic));
    ids = ids0B;
    in_blk = 0;
    i_blk = i_pos;
    ids_next = load_ids(i_blk + 32);
    ids0B = load_ids(__shfl_sync(0xffffffffu, rpB, 0));
  }
  // one commit group per call of issue(): the next edge's row if there is one, else an empty group (only after
  // the last edge of the last call, so groups and consumed rows stay in step)
  // QT > 0: ring depth known at compile time (the default 4); FULL: D == 128 * NV, no column predicate
  template <int NV, int QT = 0, bool FULL = false>
  __device__ __forceinline__ void issue() {
    const int Qc = QT > 0 ? QT : Q;
    while (i_pos == i_end && ic + 1 < ncalls) next_call();
    if (i_pos < i_end) {
      if (in_blk == 32) {
        in_blk = 0;
        i_blk += 32;
        ids = ids_next;
        ids_next = load_ids(i_blk + 32);
      }
      const int s = __shfl_sync(0xffffffffu, ids, in_blk);
      const float* rowp = h + (long long)s * ldh;
#pragma unroll
      for (int j = 0; j < NV; ++j)
        if (FULL || lane + 32 * j < C4) ptx::cp_async16(ibuf + 512u * j, rowp + 128 * j);
      ++in_blk;
      ++i_pos;
    }
    ptx::cp_async_commit();
    if (++islot == Qc) {
      islot = 0;
      ibuf = buf_s;
    } else {
      ibuf += row_bytes;
    }
  }
};

__device__ __forceinline__ void cp_async_wait_oldest(int Q) {   // at most Q-1 groups stay pending
  switch (Q) {
    case 1: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 3: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    case 4: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
    case 5: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
    case 6: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
    case 7: asm volatile("cp.async.wait_group 6;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 7;" ::: "memory"); break;
  }
}

// Tile (rank + ctas * unit) has tile_rows rows, and a ring slot as many; this warp gathers rows
// [row_off + w_row0, row_off + w_row0 + rpw) of it.
// split != 0 (split-tile mode): this CTA gathers only rows [split_rank*64, split_rank*64 + 64) of every tile; the slot
// is shared with the peer CTA of the cluster, whose slot_ready barrier gets a (cluster-scope release) arrival as well.
template <int NV, int QT = 0, bool FULL = false>
__device__ __forceinline__ void gather_warp_main(const FusedParams& p, int lane, int gw, int Q_in, uint8_t* bufs,
                                                 long long unit0, long long unit_step, long long total_units,
                                                 int ctas, int rank, int tile_rows, int row_off, int w_row0, int rpw,
                                                 int ring_row0, uint64_t* slot_ready, uint64_t* slot_free, int split,
                                                 int split_rank, uint32_t peer_slot_ready0) {
  const int Q = QT > 0 ? QT : Q_in;
  const int D = p.D, C4 = p.D >> 2, normalize = p.normalize;
  const bool no_store = p.debug_skip & 16;   // timing experiment: gathered rows are not written to the ring
  const int kFuSlots = p.num_slots;
  float* const ring = p.ring;
  const uint64_t pol_keep = ptx::policy_evict_last();
  const long long my_units = unit0 < total_units ? (total_units - unit0 + unit_step - 1) / unit_step : 0;
  GatherIssue g;
  g.row_ptr = p.row_ptr; g.src = p.src; g.h = p.h + 4 * lane; g.M = p.M; g.V = p.V; g.L = p.L; g.ldh = p.ldh;
  g.skip = p.debug_skip & 1; g.C4 = C4;
  g.lane = lane; g.gw = gw; g.Q = Q; g.ncalls = (int)(my_units * p.L);
  g.unit0 = unit0; g.unit_step = unit_step; g.ctas = ctas; g.rank = rank;
  g.tile_rows = tile_rows; g.rpw = rpw; g.row_off = row_off; g.w_row0 = w_row0;
  g.buf_s = ptx::smem_u32(bufs) + (uint32_t)lane * 16u;
  g.row_bytes = (uint32_t)p.D * 4;
  g.ic = 0; g.islot = 0; g.in_blk = 0; g.ibuf = g.buf_s;
  g.rpA = g.rp_of(0); g.rpB = g.rp_of(1); g.rpC = g.rp_of(2);
  g.i_pos = __shfl_sync(0xffffffffu, g.rpA, 0);
  g.i_end = __shfl_sync(0xffffffffu, g.rpA, g.nrows_of(0));
  g.i_blk = g.i_pos;
  g.ids = g.load_ids(g.i_blk);
  g.ids_next = g.load_ids(g.i_blk + 32);
  g.ids0B = g.load_ids(__shfl_sync(0xffffffffu, g.rpB, 0));
  // consume side: its own row_ptr registers (the issue side may already be several calls ahead after the fill)
  int crp = g.rpA, crp_next = g.rpB;
  int cslot = 0;
  uint32_t cbuf = g.buf_s;
  for (int i = 0; i < Q; ++i) g.template issue<NV, QT, FULL>();   // fill the ring

  float4 acc[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int cc = 0; cc < g.ncalls; ++cc) {
    int l, v0, nrows;
    g.call_rows(cc, l, v0, nrows);
    const int rp = crp;
    crp = crp_next;
    crp_next = g.rp_of(cc + 2);
    const int slot = cc % kFuSlots;
    if (split) ptx::mbar_wait_cluster(&slot_free[slot], ((cc / kFuSlots) & 1) ^ 1);   // the peer's reads are done too
    else ptx::mbar_wait_backoff(&slot_free[slot], ((cc / kFuSlots) & 1) ^ 1, p.sleep_long);
    float* dst = ring + ((size_t)ring_row0 + (size_t)slot * tile_rows + (size_t)row_off + (size_t)w_row0) * D + 4 * lane;
    int row = 0;
    int seg_begin = __shfl_sync(0xffffffffu, rp, 0);
    int seg_end = __shfl_sync(0xffffffffu, rp, 1);
    const int e_end = __shfl_sync(0xffffffffu, rp, nrows);
    auto flush = [&]() {   // closes row `row`
      const float scale = normalize ? 1.0f / ((float)(seg_end - seg_begin) + kSmallNumber) : 1.0f;
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        if (lane + 32 * j < C4 && !no_store)
          ptx::st_f4_hint(dst + 128 * j,
                          make_float4(acc[j].x * scale, acc[j].y * scale, acc[j].z * scale, acc[j].w * scale),
                          pol_keep);
        acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      dst += D;
      ++row;
      seg_begin = seg_end;
      seg_end = __shfl_sync(0xffffffffu, rp, row + 1);
    };
    for (int e = seg_begin; e < e_end; ++e) {
      while (e >= seg_end) flush();   // warp-uniform: close finished (possibly empty) segments
      cp_async_wait_oldest(Q);
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        if (FULL || lane + 32 * j < C4) {
          const float4 x = ptx::lds_f4(cbuf + 512u * j);
          acc[j].x += x.x; acc[j].y += x.y; acc[j].z += x.z; acc[j].w += x.w;
        }
      }
      if (++cslot == Q) {
        cslot = 0;
        cbuf = g.buf_s;
      } else {
        cbuf += g.row_bytes;
      }
      g.template issue<NV, QT, FULL>();   // refill the slot just read (same lane, same bytes: no cross-lane hazard)
    }
    while (row < nrows) flush();
    // generic-proxy global writes -> visible to the TMA (async proxy) reads of this CTA
    asm volatile("fence.proxy.async.global;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
      if (split) {   // both CTAs of the cluster read the whole slot: tell the peer's TMA producer too
        ptx::mbar_arrive_cluster_release(ptx::mapa_shared(ptx::smem_u32(&slot_ready[slot]), (uint32_t)split_rank));
        ptx::mbar_arrive_cluster_release(peer_slot_ready0 + (uint32_t)slot * 8u);
      } else {
        ptx::mbar_arrive(&slot_ready[slot]);
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Epilogue of one 64 x BN half tile (rows m0 + 64 cw + ..., columns n0 + ...) from the accumulator registers: row norm / bias /
// activation, the fused LayerNorm (single N pass: the tile holds whole rows), stores.  Thread (warp w, lane) holds rows
// 16 w + lane / 4 + {0, 8} and, of each 8-column group, columns 2 (lane % 4) + {0, 1}: a lane quad writes 32 contiguous bytes.
// FOLDED: the caller has already added the correction accumulator into the main one (the same single addition).  Only the
// row tiling folds, and it never runs the fused LayerNorm (H <= 64 keeps fused_rgcn_kernel), so that code is left out.
template <int BN, bool FOLDED = false>
__device__ __forceinline__ void fused_epilogue(const FusedParams& p, const HalfTileAcc<BN>& c, long long m0, int n0, int cw,
                                               int t) {
  const int w = t >> 5, lane = t & 31, cq = 2 * (lane & 3);
  const uint64_t pol_stream = ptx::policy_evict_first();
  const bool ln = !FOLDED && p.epi.ln_gamma != nullptr;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = m0 + 64 * cw + 16 * w + (lane >> 2) + 8 * h;
    const bool row_ok = row < p.V;
    float v[BN / 4];
    if (FOLDED) {
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        v[2 * i] = c.main[4 * i + 2 * h];
        v[2 * i + 1] = c.main[4 * i + 2 * h + 1];
      }
    } else {
      acc_row<BN>(c, h, v);
    }
    if (p.epi.row_norm && row_ok) {
      const float inv_rn = 1.0f / fu_row_norm(p.epi, row);
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) v[j] *= inv_rn;
    }
    if (p.epi.bias) {
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.epi.bias + n0 + 8 * i + cq));
        v[2 * i] += b.x; v[2 * i + 1] += b.y;
      }
    }
    apply_act_vec<BN / 4>(v, p.epi.act);
    if (ln) {
      // LayerNormalization over the finished row (gnn.py:317-321 right after the message-passing layer): the quad holds the
      // row; two-pass variance (mean first) like Keras
      float s1 = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) s1 += v[j];
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      const float mean = s1 / (float)BN;
      float s2 = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) { const float d = v[j] - mean; s2 = fmaf(d, d, s2); }
      s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
      s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
      const float rstd = rsqrtf(s2 / (float)BN + p.epi.ln_eps);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const float2 g = __ldg(reinterpret_cast<const float2*>(p.epi.ln_gamma + n0 + 8 * i + cq));
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.epi.ln_beta + n0 + 8 * i + cq));
        v[2 * i] = (v[2 * i] - mean) * rstd * g.x + b.x;
        v[2 * i + 1] = (v[2 * i + 1] - mean) * rstd * g.y + b.y;
      }
    }
    if (!row_ok) continue;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const long long off = row * p.ldc + n0 + 8 * i + cq;
      const float2 val = make_float2(v[2 * i], v[2 * i + 1]);
      if (p.C_mc) {
        // the all-gather of the sharded layer through the switch: ONE multimem.st, NVSwitch replicates the 8 bytes into every
        // GPU's copy of the table (this GPU's included)
        asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(p.C_mc + off), "f"(val.x), "f"(val.y)
                     : "memory");
      } else {
        asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p.C + off), "f"(val.x), "f"(val.y),
                     "l"(pol_stream)
                     : "memory");
        // the all-gather of the sharded layer, tile by tile: the same bytes go to every peer's copy of the table over NVLink
        // (plain stores to P2P-mapped memory; the copies become the next layer's source table)
        for (int pr = 0; pr < p.n_peer; ++pr) *reinterpret_cast<float2*>(p.C_peer[pr] + off) = val;
      }
    }
  }
}

// SPLIT (small batches, fewer than SMs/2 tiles): the two CTAs of a cluster share ONE 128-target tile.  Each gathers half of
// its rows into the common ring slot and contracts the whole tile with its HALF of the output columns: the gather (bound by
// one SM's L2 bandwidth when a tile is all an SM has) and the K loop are both spread over twice as many SMs.  Ring slots are
// released only when both CTAs have read them.
template <int NV, int BN>
__global__ void __launch_bounds__(kFuThreads, 1)
fused_rgcn_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const FusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int b_tile_bytes = BN * kFuBK * 4;
  constexpr int stage_bytes = 2 * kFuATileBytes + 2 * b_tile_bytes;
  const int S = p.num_stages;
  const bool split = p.split != 0;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes);
  uint64_t* full = bars;                          // TMA bytes landed
  uint64_t* empty = bars + S;                     // both consumer warpgroups' MMAs reading the stage retired
  uint64_t* slot_ready = bars + 2 * S;
  uint64_t* slot_free = bars + 2 * S + kFuMaxSlots;
  uint8_t* gbuf = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(bars + 2 * S + 2 * kFuMaxSlots) + 127) & ~uintptr_t(127));   // [8 * Q] rows

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const uint32_t srank = split ? ptx::cluster_ctarank() : 0u;   // split-tile mode: which half (rows to gather, columns to produce)
  const int kClu = split ? 2 : 1;                                // CTAs per cluster
  // one unit = one 128-target tile; the CTA's cta_n columns are covered in n_pass passes of BN
  const long long total_units = p.m_tiles;
  const long long unit0 = blockIdx.x / kClu, unit_step = gridDim.x / kClu;
  const int n_pass = p.n_tiles;
  const int kFuSlots = p.num_slots;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&map_a);
    ptx::prefetch_tensormap(&map_b);
    for (int s = 0; s < S; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 2);
    }
    for (int r = 0; r < kFuMaxSlots; ++r) {
      ptx::mbar_init(&slot_ready[r], kFuGatherWarps * (split ? 2 : 1));   // split: the peer's gather warps arrive too
      ptx::mbar_init(&slot_free[r], 2 * (split ? 2 : 1));                 // one arrival per consumer warpgroup (of both CTAs)
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (split) ptx::cluster_sync_all();   // both CTAs' barriers exist before any remote arrive can land on them
  // first ring row of this CTA (split-tile mode: of this CLUSTER, both CTAs fill and read the same slots)
  const int ring_row0 = (split ? blockIdx.x / 2 : blockIdx.x) * kFuSlots * kFuBM;
  const uint32_t peer_slot_ready0 = split ? ptx::mapa_shared(ptx::smem_u32(&slot_ready[0]), srank ^ 1u) : 0u;
  const uint32_t peer_slot_free0 = split ? ptx::mapa_shared(ptx::smem_u32(&slot_free[0]), srank ^ 1u) : 0u;

  if (warp == 8) {
    // ================= TMA producer =================
    if (lane == 0) {
      uint32_t it = 0, slot_it = 0;
      const uint64_t pol_keep = ptx::policy_evict_last();   // ring slots and the weights stay in L2
      for (long long unit = unit0; unit < total_units; unit += unit_step, slot_it += p.L) {
        for (int pass = 0; pass < n_pass; ++pass) {
          const int n0 = (int)srank * p.cta_n + pass * BN;
          for (int l = 0; l < p.L; ++l) {
            const uint32_t sq = slot_it + l;
            const int slot = sq % kFuSlots;
            if (split) ptx::mbar_wait_cluster(&slot_ready[slot], (sq / kFuSlots) & 1);   // half of the rows come from the peer SM
            else ptx::mbar_wait_backoff(&slot_ready[slot], (sq / kFuSlots) & 1, p.sleep_long);
            for (int kb = 0; kb < p.kb_per_type; ++kb, ++it) {
              const int s = it % S;
              const uint32_t ph = (it / S) & 1;
              ptx::mbar_wait_backoff(&empty[s], ph ^ 1, p.sleep_crit);
              uint8_t* st = smem + (size_t)s * stage_bytes;
              ptx::mbar_arrive_expect_tx(&full[s], kFuATileBytes + 2 * b_tile_bytes);
              ptx::tma_load_2d_hint(st, &map_a, &full[s], kb * kFuBK, ring_row0 + slot * kFuBM, pol_keep);
              const int kcol = (l * p.kb_per_type + kb) * kFuBK;
              ptx::tma_load_2d_hint(st + 2 * kFuATileBytes, &map_b, &full[s], kcol, n0, pol_keep);
              ptx::tma_load_2d_hint(st + 2 * kFuATileBytes + b_tile_bytes, &map_b, &full[s], kcol, p.N + n0, pol_keep);
            }
          }
        }
      }
    }
  } else if (wg < 2) {
    // ================= consumers: warpgroups 0, 1 -> rows [0, 64), [64, 128) of every tile =================
    const int cw = wg, t = threadIdx.x & 127;
    HalfTileAcc<BN> c;
    uint32_t it = 0, slot_base_it = 0;
    for (long long unit = unit0; unit < total_units; unit += unit_step, slot_base_it += p.L) {
      for (int pass = 0; pass < n_pass; ++pass) {
        int prev_s = 0;
        bool first = true;
        for (int l = 0; l < p.L; ++l) {
          const uint32_t slot_it = slot_base_it + l;
          for (int kb = 0; kb < p.kb_per_type; ++kb, ++it) {
            const int s = it % S;
            const uint32_t ph = (it / S) & 1;
            ptx::mbar_wait_backoff(&full[s], ph, p.sleep_crit);
            // all TMA reads of the slot have landed: its lines are dead.  Discard this warpgroup's rows from L2 so that they
            // are never written back to HBM (the ring is pure on-chip hand-off), then hand the slot back.
            const bool slot_done = kb == p.kb_per_type - 1 && pass == n_pass - 1;
            if (slot_done && p.discard_ring && !split) {   // split-tile mode: the peer may still be reading the slot
              const char* sb = reinterpret_cast<const char*>(
                  p.ring + ((size_t)ring_row0 + (size_t)(slot_it % kFuSlots) * kFuBM + (size_t)cw * 64) * p.D);
              const int lines = 64 * p.D * 4 / 128;
              for (int i = t; i < lines; i += 128) ptx::discard_l2_128(sb + (size_t)i * 128);
            }
            const uint32_t st = ptx::smem_u32(smem + (size_t)s * stage_bytes);
            split_a_half<128>(st, cw, t, p.corr_bf16);
            ptx::fence_proxy_async_smem();
            ptx::warpgroup_sync(1 + cw);
            if (slot_done && t == 0) {
              ptx::mbar_arrive(&slot_free[slot_it % kFuSlots]);
              if (split) ptx::mbar_arrive_cluster_release(peer_slot_free0 + (uint32_t)(slot_it % kFuSlots) * 8u);
            }
            ptx::wgmma_fence();
            mma_kblock<BN, 128>(c, st, st + 2 * kFuATileBytes, cw, p.corr_bf16, first);
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();   // the previous block's MMAs are done: its stage goes back to the producer
            if (!first && t == 0) ptx::mbar_arrive(&empty[prev_s]);
            prev_s = s;
            first = false;
          }
        }
        ptx::wgmma_wait<0>();
        fence_acc<BN>(c);
        if (t == 0) ptx::mbar_arrive(&empty[prev_s]);
        fused_epilogue<BN>(p, c, unit * kFuBM, (int)srank * p.cta_n + pass * BN, cw, t);
      }
    }
  } else {
    // ================= gather warps =================
    const int gw = warp - kFuFirstGatherWarp;
    // common case (ring depth 8, D a multiple of 128): depth and column predicate resolved at compile time - the gather
    // loop runs once per EDGE
    uint8_t* my_bufs = gbuf + (size_t)gw * p.gather_q * ((size_t)p.D * 4);
    const int rpw = split ? kFuBM / 2 / kFuGatherWarps : kFuBM / kFuGatherWarps;
    const int row_off = split ? (int)srank * (kFuBM / 2) : 0;
#define TFGNN_FU_GATHER(QT, FULL)                                                                                     \
    gather_warp_main<NV, QT, FULL>(p, lane, gw, p.gather_q, my_bufs, unit0, unit_step, total_units, 1, 0, kFuBM,       \
                                   row_off, gw * rpw, rpw, ring_row0, slot_ready, slot_free, split ? 1 : 0, (int)srank, \
                                   peer_slot_ready0)
    if (p.gather_q == kFuMaxQ && p.D == 128 * NV) TFGNN_FU_GATHER(kFuMaxQ, true);
    else TFGNN_FU_GATHER(0, false);
#undef TFGNN_FU_GATHER
  }

  if (split) {
    __syncwarp();
    ptx::cluster_sync_all();   // remote arrivals target the peer's shared memory: leave together
  }
}

// ---- row tiling (64 < H <= 256, H % 32 == 0): the N dimension in ONE pass ------------------------------------------------
// The two CTAs of a cluster share each 128-row x H tile ("unit"), split by columns: CTA r gathers rows [64 r, 64 r + 64) of
// the unit into its own ring slot (64 rows, one edge type) and produces columns [r BN, r BN + BN) of all 128 rows, BN = H / 2.
// For every K block each producer loads its 64 ring rows once and multicasts them into both CTAs' stage (at row 64 r of a
// 128-row A tile), and loads only its own BN columns of the pre-split weights.  So an SM receives 16 KB of A and 2 BN x 128 B
// of weights per K block (48 KB at H = 256), and each weight byte it receives serves 128 rows.  Consumer warpgroup w splits
// rows [64 w, 64 w + 64) of A and contracts them with this CTA's BN columns (main + correction: BN registers per thread, 128
// at H = 256).  The registers come from setmaxnreg: the kernel launches at 128 per thread (512 threads) and the TMA / gather
// warpgroups hand theirs to the consumers.  A ring slot is released as soon as its last K block has landed, so the gather
// runs up to a whole unit ahead of the MMAs.  Both CTAs walk the same (type, K block) sequence in lockstep: every stage is
// written by both producers, so it is refilled once all four consumer warpgroups of the pair have released it.  With an odd
// 64-row tile count the last cluster's second CTA gathers an empty tile; both CTAs still store their columns of the first
// 64 rows.  The K order of every output element (type, K block, k8 step; main and correction added in the epilogue) is that
// of fused_rgcn_kernel, so both give the same bits.
//
// Warp roles (512 threads, warpgroup-aligned):
//   0-7: two consumer warpgroups | 8: TMA | 9-15: gather (64 / 7 rows each: 9 or 10).
constexpr int kRtBM = 64;
constexpr int kRtATileBytes = kRtBM * kFuBK * 4;
constexpr int kRtGatherWarps = 7;
constexpr int kRtFirstGatherWarp = 9;
constexpr int kRtThreads = 512;
constexpr int kRtMaxH = 256;
constexpr uint32_t kRtConsumerRegs = 184;   // + kRtOtherRegs = 256: the register file at 512 threads
constexpr uint32_t kRtOtherRegs = 72;

template <int NV, int BN>
__global__ void __launch_bounds__(kRtThreads, 1)
fused_rgcn_rows_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                       const FusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int H = 2 * BN;
  constexpr int b_tile_bytes = BN * kFuBK * 4;    // this CTA's columns of one weight half (hi or correction)
  constexpr int stage_bytes = 2 * kFuATileBytes + 2 * b_tile_bytes;
  const int S = p.num_stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes);
  uint64_t* full = bars;                          // both CTAs' rows of A and this CTA's weights landed
  uint64_t* empty = bars + S;                     // the MMAs of all four consumer warpgroups of the cluster retired
  uint64_t* slot_ready = bars + 2 * S;
  uint64_t* slot_free = bars + 2 * S + kFuMaxSlots;
  uint8_t* gbuf = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(bars + 2 * S + 2 * kFuMaxSlots) + 127) & ~uintptr_t(127));   // [7 * Q] rows

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const uint32_t srank = ptx::cluster_ctarank();
  // one unit = the cluster's 128-row tile; this CTA gathers its 64-row tile 2 unit + srank
  const long long total_units = (p.m_tiles + 1) / 2;
  const long long unit0 = blockIdx.x / 2, unit_step = gridDim.x / 2;
  const int kSlots = p.num_slots;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&map_a);
    ptx::prefetch_tensormap(&map_b);
    for (int s = 0; s < S; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 4);
    }
    for (int r = 0; r < kFuMaxSlots; ++r) {
      ptx::mbar_init(&slot_ready[r], kRtGatherWarps);
      ptx::mbar_init(&slot_free[r], 2);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::cluster_sync_all();   // both CTAs' barriers exist before any multicast or remote arrive can land on them
  const int ring_row0 = blockIdx.x * kSlots * kRtBM;

  if (wg >= 2) {
    ptx::setmaxnreg_dec<kRtOtherRegs>();
    if (warp == 8) {
      // ================= TMA producer =================
      if (lane == 0) {
        uint32_t it = 0, slot_it = 0;
        const uint64_t pol_keep = ptx::policy_evict_last();   // ring slots and the weights stay in L2
        for (long long unit = unit0; unit < total_units; unit += unit_step, slot_it += p.L) {
          for (int l = 0; l < p.L; ++l) {
            const uint32_t sq = slot_it + l;
            const int slot = sq % kSlots;
            ptx::mbar_wait_backoff(&slot_ready[slot], (sq / kSlots) & 1, p.sleep_long);
            for (int kb = 0; kb < p.kb_per_type; ++kb, ++it) {
              const int s = it % S;
              const uint32_t ph = (it / S) & 1;
              // both CTAs' copies of the stage are free (the multicast below writes into the peer's as well)
              ptx::mbar_wait_cluster(&empty[s], ph ^ 1);
              uint8_t* st = smem + (size_t)s * stage_bytes;
              // this CTA's full[s] counts both producers' rows of A and its own weight columns
              ptx::mbar_arrive_expect_tx(&full[s], kFuATileBytes + 2 * b_tile_bytes);
              ptx::tma_load_2d_multicast_hint(st + (int)srank * kRtATileBytes, &map_a, &full[s], kb * kFuBK,
                                              ring_row0 + slot * kRtBM, (uint16_t)0x3, pol_keep);
              const int kcol = (l * p.kb_per_type + kb) * kFuBK;
              ptx::tma_load_2d_hint(st + 2 * kFuATileBytes, &map_b, &full[s], kcol, (int)srank * BN, pol_keep);
              ptx::tma_load_2d_hint(st + 2 * kFuATileBytes + b_tile_bytes, &map_b, &full[s], kcol, H + (int)srank * BN,
                                    pol_keep);
            }
          }
        }
      }
    } else {
      // ================= gather warps =================
      const int gw = warp - kRtFirstGatherWarp;
      const int w_row0 = kRtBM * gw / kRtGatherWarps, rpw = kRtBM * (gw + 1) / kRtGatherWarps - w_row0;
      uint8_t* my_bufs = gbuf + (size_t)gw * p.gather_q * ((size_t)p.D * 4);
#define TFGNN_RT_GATHER(QT, FULL)                                                                                      \
      gather_warp_main<NV, QT, FULL>(p, lane, gw, p.gather_q, my_bufs, unit0, unit_step, total_units, 2, (int)srank,   \
                                     kRtBM, 0, w_row0, rpw, ring_row0, slot_ready, slot_free, 0, 0, 0u)
      if (p.gather_q == kFuMaxQ && p.D == 128 * NV) TFGNN_RT_GATHER(kFuMaxQ, true);
      else TFGNN_RT_GATHER(0, false);
#undef TFGNN_RT_GATHER
    }
  } else {
    // ================= consumers: warpgroup cw -> rows [64 cw, 64 cw + 64) x this CTA's BN columns =================
    ptx::setmaxnreg_inc<kRtConsumerRegs>();
    const int cw = wg, t = threadIdx.x & 127;
    const uint32_t empty0_cta0 = ptx::mapa_shared(ptx::smem_u32(&empty[0]), 0u);
    const uint32_t empty0_cta1 = ptx::mapa_shared(ptx::smem_u32(&empty[0]), 1u);
    // One arrival per consumer warpgroup on the stage's barrier in BOTH CTAs.  A plain arrive: the stage's only readers are
    // this warpgroup's retired MMAs (wgmma.wait_group 0), and its split stores were read by them, so nothing is left for a
    // cluster-scope release to order before the producers' refill.  The release form costs a GPU-scope memory barrier per
    // arrive (MEMBAR.ALL.GPU), which also waits for the epilogue stores and L2 discards still in flight.
    auto release_stage = [&](int s) {
      if (t == 0) {
        ptx::mbar_arrive_cluster(empty0_cta0 + (uint32_t)s * 8u);
        ptx::mbar_arrive_cluster(empty0_cta1 + (uint32_t)s * 8u);
      }
    };
    HalfTileAcc<BN> c;
    uint32_t it = 0, slot_base_it = 0;
    for (long long unit = unit0; unit < total_units; unit += unit_step, slot_base_it += p.L) {
      bool first = true;
      for (int l = 0; l < p.L; ++l) {
        const int slot = (slot_base_it + l) % kSlots;
        for (int kb = 0; kb < p.kb_per_type; ++kb, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          ptx::mbar_wait_backoff(&full[s], ph, p.sleep_crit);
          // The last K block of this CTA's slot has landed here, and only this CTA's producer reads the slot (the peer gets
          // the rows through the multicast, from the same L2 read): its lines are dead.  This warpgroup discards half of the
          // rows from L2 (never written back to HBM), and the slot goes back to the gather warps.  Split-tile mode
          // (fused_rgcn_kernel) cannot discard, because there the peer CTA reads the shared slot itself.
          const bool slot_done = kb == p.kb_per_type - 1;
          if (slot_done && p.discard_ring) {
            const char* sb = reinterpret_cast<const char*>(
                p.ring + ((size_t)ring_row0 + (size_t)slot * kRtBM + (size_t)cw * (kRtBM / 2)) * p.D);
            const int lines = kRtBM / 2 * p.D * 4 / 128;
            for (int i = t; i < lines; i += 128) ptx::discard_l2_128(sb + (size_t)i * 128);
          }
          const uint32_t st = ptx::smem_u32(smem + (size_t)s * stage_bytes);
          split_a_half<128>(st, cw, t, p.corr_bf16);   // this warpgroup's 64 rows only
          ptx::fence_proxy_async_smem();
          ptx::warpgroup_sync(1 + cw);
          if (slot_done && t == 0) ptx::mbar_arrive(&slot_free[slot]);
          ptx::wgmma_fence();
          mma_kblock<BN, 128>(c, st, st + 2 * kFuATileBytes, cw, p.corr_bf16, first);
          ptx::wgmma_commit();
          // The stage goes back to both producers as soon as its MMAs retire, before the next stage is waited for.  On cfg2
          // this measured as fast as three stages (gather depth 4 instead of 8) that keep one K block of MMAs in flight.
          ptx::wgmma_wait<0>();
          release_stage(s);
          first = false;
        }
      }
      fence_acc<BN>(c);
      // main + correction first: the correction registers are free for the epilogue
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) c.main[j] += c.corr[j];
      // rows past V (the second half of the last unit with an odd tile count: all of them) are not stored.  The warpgroup's
      // row offset goes into m0 (cw = 0) so that the epilogue needs no extra register for it.
      fused_epilogue<BN, true>(p, c, unit * kFuBM + 64 * cw, (int)srank * BN, 0, t);
    }
  }
  __syncwarp();
  ptx::cluster_sync_all();   // multicasts and remote arrivals target the peer's shared memory: leave together
}

// ---- host side -------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn fu_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// Column tile of the fused kernel for n output columns per CTA: the widest multiple of 16 (<= kFuMaxBN) that divides n.
static int fused_block_n(int n) {
  for (int bn = kFuMaxBN; bn >= 16; bn -= 16)
    if (n % bn == 0) return bn;
  return 0;
}

bool fused_rgcn_supported(long long V, int L, int D, int H, const float* h, const float* out, int ldo) {
  if (V < 1 || L < 1 || D % 32 != 0 || D > 512 || H % 16 != 0 || H < 16 || H > 512) return false;
  if (fused_block_n(H) < H && L + 1 > kFuMaxSlots) return false;   // several N passes: the ring holds L+1 slots
  if ((reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(out)) & 15) return false;
  if (ldo % 4 != 0) return false;
  // every source row is gathered exactly once; H > 128 takes several passes over the ring
  return gemm_tc_supported(V, H, L * D, h, D, out, ldo) && fu_encode_fn() != nullptr;
}

bool fused_rgcn_ln_supported(int H) { return H <= kFuMaxBN; }

// ---- device-global state: the persisting-L2 carve-out ---------------------------------------------------------
// cudaLimitPersistingL2CacheSize is a property of the DEVICE CONTEXT the host framework shares with this library, so
// it is handled explicitly (include/tfgnn_b200.h, "Device-global state"): the first fused launch on a device saves
// the current limit and raises it to the configured size (default: ring + packed weights, clamped to the device's
// maximum set-aside); tfgnn_b200_set_l2_persist_mb(0) / TFGNN_B200_L2_PERSIST_MB=0 opt out (the kernel stays correct,
// the ring is then written back to HBM); tfgnn_b200_release_device_state() restores the saved limit.
static std::mutex g_l2_mu;
static int g_l2_want_mb = -1;                 // -1: default / environment
static bool g_l2_set[64] = {};
static size_t g_l2_saved[64] = {};

int set_l2_persist_mb(int mb) {
  std::lock_guard<std::mutex> lock(g_l2_mu);
  g_l2_want_mb = mb;
  for (bool& b : g_l2_set) b = false;         // re-applied by the next fused launch
  return 0;
}

static size_t g_l2_effective[64] = {};   // persisting bytes in effect on the device since the last ensure()

// need_bytes: what this launch wants resident (its ring + packed weights).  Default policy: max(72 MB, need + 4 MB), clamped
// to the device maximum and only ever RAISED; an explicit size (API / environment) is taken as is.
static int ensure_l2_persist_carveout(size_t need_bytes) {
  int dev = 0;
  TFGNN_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return 0;
  std::lock_guard<std::mutex> lock(g_l2_mu);
  long long want_mb = g_l2_want_mb;
  if (want_mb < 0) {
    static const int env_mb = [] { const char* e = getenv("TFGNN_B200_L2_PERSIST_MB"); return e ? atoi(e) : -1; }();
    want_mb = env_mb;
  }
  size_t want = want_mb >= 0 ? (size_t)want_mb << 20 : std::max((size_t)72 << 20, need_bytes + ((size_t)4 << 20));
  if (g_l2_set[dev] && (want_mb >= 0 || g_l2_effective[dev] >= want)) return 0;
  g_l2_set[dev] = true;
  if (want == 0) return 0;
  int max_persist = 0;
  if (cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev) != cudaSuccess || max_persist <= 0) {
    cudaGetLastError();
    return 0;
  }
  if (want > (size_t)max_persist) want = (size_t)max_persist;
  size_t cur = 0;
  if (cudaDeviceGetLimit(&cur, cudaLimitPersistingL2CacheSize) != cudaSuccess) { cudaGetLastError(); return 0; }
  g_l2_effective[dev] = cur;
  if (cur >= want) {                          // the host (or an earlier launch) already reserves at least as much
    if (want == (size_t)max_persist) g_l2_effective[dev] = (size_t)-1;   // nothing more to get: stop asking
    return 0;
  }
  if (!g_l2_saved[dev]) g_l2_saved[dev] = cur + 1;   // +1: "saved" marker (0 = nothing to restore)
  cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want);
  cudaGetLastError();
  g_l2_effective[dev] = want == (size_t)max_persist ? (size_t)-1 : want;
  return 0;
}

void restore_l2_persist_carveout() {
  std::lock_guard<std::mutex> lock(g_l2_mu);
  int cur_dev = 0;
  if (cudaGetDevice(&cur_dev) != cudaSuccess) { cudaGetLastError(); return; }
  for (int d = 0; d < 64; ++d) {
    if (!g_l2_saved[d]) continue;
    if (cudaSetDevice(d) == cudaSuccess) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, g_l2_saved[d] - 1);
    g_l2_saved[d] = 0;
    g_l2_set[d] = false;
    g_l2_effective[d] = 0;
  }
  cudaSetDevice(cur_dev);
  cudaGetLastError();
}

constexpr int kFuMaxGrid = 160;
// Row tiling: 3 slots of 64 rows by default (26 MB of ring at D = 256 on 132 SMs).  On cfg2 (H100 SXM, 400 W) 2 slots ran
// within 1 % of 3, and 4 and 5 slots 6 % and 13 % slower (DESIGN.md §4): the smaller ring leaves more of L2 to the weights
// and the source rows.
static int fused_num_slots(int L, bool multi_pass, bool rows = false) {
  static const int env_slots = [] { const char* e = getenv("TFGNN_B200_RING_SLOTS"); return e ? atoi(e) : 0; }();
  if (multi_pass) return L + 1;
  return (env_slots >= 2 && env_slots <= kFuMaxSlots) ? env_slots : rows ? 3 : 4;
}
size_t fused_rgcn_ring_bytes(int D, int L, int H) {
  (void)H;   // covers every tiling (single or several N passes, split-tile mode; the row tiling's 64-row slots need half)
  int slots = fused_num_slots(L, false);
  if (L + 1 <= kFuMaxSlots && L + 1 > slots) slots = L + 1;
  return (size_t)kFuMaxGrid * slots * kFuBM * D * sizeof(float);
}

template <int NV, int BN>
static cudaError_t launch_fused_nv_bn(cudaLaunchConfig_t& cfg, const CUtensorMap& map_a, const CUtensorMap& map_b,
                                      const FusedParams& p) {
  static std::once_flag attr_once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once, [] {
    attr_err = cudaFuncSetAttribute(fused_rgcn_kernel<NV, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmemLimit);
  });
  if (attr_err != cudaSuccess) return attr_err;
  return cudaLaunchKernelEx(&cfg, fused_rgcn_kernel<NV, BN>, map_a, map_b, p);
}

template <int NV>
static cudaError_t launch_fused_nv(cudaLaunchConfig_t& cfg, const CUtensorMap& map_a, const CUtensorMap& map_b,
                                   const FusedParams& p) {
  switch (p.block_n) {
    case 16: return launch_fused_nv_bn<NV, 16>(cfg, map_a, map_b, p);
    case 32: return launch_fused_nv_bn<NV, 32>(cfg, map_a, map_b, p);
    case 48: return launch_fused_nv_bn<NV, 48>(cfg, map_a, map_b, p);
    default: return launch_fused_nv_bn<NV, 64>(cfg, map_a, map_b, p);
  }
}

// Row tiling: clusters of 2 CTAs, each a whole SM; the grid is sized to the clusters that can be resident at once (the
// kernel is persistent: a cluster that has to wait for a free SM pair would run its tiles after everybody else's).
template <int NV, int BN>
static cudaError_t launch_fused_rows_nv_bn(cudaLaunchConfig_t& cfg, const CUtensorMap& map_a, const CUtensorMap& map_b,
                                           const FusedParams& p, long long units, int max_clusters) {
  static std::mutex mu;
  static cudaError_t attr_err = cudaSuccess;
  static bool attr_set = false;
  static size_t occ_smem = 0;
  static int occ_clusters = 0;
  int clusters = 0;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (!attr_set) {
      attr_err = cudaFuncSetAttribute(fused_rgcn_rows_kernel<NV, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kFuSmemLimit);
      attr_set = true;
    }
    if (attr_err != cudaSuccess) return attr_err;
    if (occ_smem != cfg.dynamicSmemBytes) {
      cfg.gridDim = dim3(2u * (unsigned)max_clusters);
      int n = 0;
      cudaError_t e = cudaOccupancyMaxActiveClusters(&n, fused_rgcn_rows_kernel<NV, BN>, &cfg);
      if (e != cudaSuccess) return e;
      if (n < 1) return cudaErrorInvalidConfiguration;
      occ_smem = cfg.dynamicSmemBytes;
      occ_clusters = n;
    }
    clusters = std::min(occ_clusters, max_clusters);
  }
  if (units < clusters) clusters = (int)units;
  cfg.gridDim = dim3(2u * (unsigned)clusters);
  return cudaLaunchKernelEx(&cfg, fused_rgcn_rows_kernel<NV, BN>, map_a, map_b, p);
}

template <int NV>
static cudaError_t launch_fused_rows_nv(cudaLaunchConfig_t& cfg, const CUtensorMap& map_a, const CUtensorMap& map_b,
                                        const FusedParams& p, long long units, int max_clusters) {
  switch (p.block_n) {
    case 48: return launch_fused_rows_nv_bn<NV, 48>(cfg, map_a, map_b, p, units, max_clusters);
    case 64: return launch_fused_rows_nv_bn<NV, 64>(cfg, map_a, map_b, p, units, max_clusters);
    case 80: return launch_fused_rows_nv_bn<NV, 80>(cfg, map_a, map_b, p, units, max_clusters);
    case 96: return launch_fused_rows_nv_bn<NV, 96>(cfg, map_a, map_b, p, units, max_clusters);
    case 112: return launch_fused_rows_nv_bn<NV, 112>(cfg, map_a, map_b, p, units, max_clusters);
    default: return launch_fused_rows_nv_bn<NV, 128>(cfg, map_a, map_b, p, units, max_clusters);
  }
}

int launch_fused_rgcn(const float* h, int D, const int* row_ptr, const int* src, long long M, int V, int L,
                      int normalize, const float* packedB, int corr_bf16, int H, float* ring, float* out, int ldo,
                      const GemmEpilogue& epi, cudaStream_t st, float* const* peer_out, int n_peer_out, float* mc_out) {
  EncodeTiledFn encode = fu_encode_fn();
  if (!encode) {
    set_error(TFGNN_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    return TFGNN_ERR_CUDA;
  }
  int dev = 0, sms = 0;
  TFGNN_CUDA(cudaGetDevice(&dev));
  TFGNN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  FusedParams p{};
  p.h = h; p.ldh = D; p.row_ptr = row_ptr; p.src = src; p.V = V; p.L = L; p.D = D; p.normalize = normalize;
  p.ring = ring;
  p.M = M;
  static const int discard_env = [] { const char* e = getenv("TFGNN_B200_RING_DISCARD"); return e ? atoi(e) : 1; }();
  p.discard_ring = discard_env;
  static const int dbg_env = [] { const char* e = getenv("TFGNN_B200_DEBUG_SKIP"); return e ? atoi(e) : 0; }();
  p.debug_skip = dbg_env;
  p.corr_bf16 = corr_bf16;
  p.n_peer = 0;
  for (int r = 0; r < n_peer_out && r < TFGNN_MAX_PEERS; ++r) p.C_peer[p.n_peer++] = peer_out[r];
  p.C_mc = mc_out;
  p.N = H;
  p.m_tiles = ((long long)V + kFuBM - 1) / kFuBM;
  if (sms > kFuMaxGrid) sms = kFuMaxGrid;
  const bool want_ln = epi.ln_gamma != nullptr;   // the row statistics need the whole row in one CTA: single N pass, no split
  TFGNN_REQUIRE(!want_ln || fused_rgcn_ln_supported(H), "fused LayerNorm needs hidden_dim <= 64 (one N pass)");
  // Split-tile mode (small batches): fewer tiles than half the SMs -> two CTAs share each tile (rows of the gather,
  // columns of the contraction).  TFGNN_B200_FUSED_SPLIT: 0 = never, 1 = default rule (read per call: the tests sweep it)
  const char* split_str = getenv("TFGNN_B200_FUSED_SPLIT");
  const int split_env = split_str ? atoi(split_str) : 1;
  const bool split = !want_ln && split_env != 0 && 2 * p.m_tiles <= sms && H % 32 == 0 &&
                     (fused_block_n(H / 2) == H / 2 || L + 1 <= kFuMaxSlots);
  // Row tiling (fused_rgcn_rows_kernel): 128 x H tiles in one N pass, split by columns over a CTA pair (m_tiles counts the
  // 64-row halves each CTA gathers), for the full-size launch of the layers wider than one
  // 64-column tile up to H = 256.  Split-tile mode, the fused LayerNorm (H <= 64) and H > 256 keep fused_rgcn_kernel.
  const bool rows = !split && !want_ln && H > kFuMaxBN && H <= kRtMaxH && H % 32 == 0;
  p.split = split ? 1 : 0;
  p.cta_n = split ? H / 2 : H;
  p.block_n = rows ? H / 2 : fused_block_n(p.cta_n);   // row tiling: the columns of one consumer warpgroup
  p.n_tiles = rows ? 1 : p.cta_n / p.block_n;          // N passes (per CTA)
  p.num_slots = fused_num_slots(L, p.n_tiles > 1, rows);
  const int tile_rows = rows ? kRtBM : kFuBM;
  if (rows) p.m_tiles = ((long long)V + kRtBM - 1) / kRtBM;
  p.C = out; p.ldc = ldo; p.epi = epi;
  {
    const char* sc = getenv("TFGNN_B200_SLEEP_CRIT");
    const char* sl = getenv("TFGNN_B200_SLEEP_LONG");
    p.sleep_crit = sc ? (uint32_t)atoi(sc) : 0u;
    p.sleep_long = sl ? (uint32_t)atoi(sl) : 0u;
  }
  // row tiling: the largest grid (the launch may shrink it to the co-resident clusters); it sizes the ring's tensor map
  const int grid = rows ? (sms & ~1)
                 : split ? (int)(2 * p.m_tiles < (sms & ~1) ? 2 * p.m_tiles : (sms & ~1)) : (int)(p.m_tiles < sms ? p.m_tiles : sms);
  // shared memory: S pipeline stages + Q row slots for each gather warp.  The gather gets its Q rows in flight first (8 per
  // warp: as many bytes in flight as 16 warps x 4); the pipeline gets what is left (2..4 stages).
  static const int stage_env = [] { const char* e = getenv("TFGNN_B200_FUSED_STAGES"); return e ? atoi(e) : 0; }();
  const char* q_str = getenv("TFGNN_B200_GATHER_Q");   // read per call: the tests sweep it
  const int q_env = q_str ? atoi(q_str) : 0;
  const int fixed_bytes = 2048 + 128 + 1024;   // barriers, alignment slack
  const int row_bytes = D * 4;
  const int want_q = q_env >= 1 && q_env <= kFuMaxQ ? q_env : kFuMaxQ;
  const int gather_warps = rows ? kRtGatherWarps : kFuGatherWarps;
  // A and its correction operand (128 rows each) + the hi and correction rows of the CTA's block_n weight columns
  const int stage_bytes = 2 * kFuATileBytes + 2 * p.block_n * kFuBK * 4;
  auto q_for = [&](int s_) { return (kFuSmemLimit - fixed_bytes - s_ * stage_bytes) / (gather_warps * row_bytes); };
  int stages = stage_env >= 2 ? stage_env : 4;
  while (stages > 2 && q_for(stages) < want_q) --stages;
  int q = q_for(stages);
  if (q > want_q) q = want_q;
  TFGNN_REQUIRE(q >= 1 && stages >= 2, "fused RGCN: tile does not fit shared memory");
  p.kb_per_type = D / kFuBK;
  if (p.debug_skip & 2) p.kb_per_type = 1;
  p.num_stages = stages;
  p.gather_q = q;

  const int Kp = L * D;
  CUtensorMap map_a, map_b;
  {
    cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)grid * p.num_slots * tile_rows};
    cuuint64_t strides[1] = {(cuuint64_t)D * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)kFuBK, (cuuint32_t)tile_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(&map_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ring, dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error(TFGNN_ERR_CUDA, "cuTensorMapEncodeTiled(ring) failed with code " + std::to_string((int)r));
      return TFGNN_ERR_CUDA;
    }
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)(2 * H)};
    cuuint64_t strides[1] = {(cuuint64_t)Kp * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)kFuBK, (cuuint32_t)p.block_n};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(&map_b, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(packedB), dims, strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error(TFGNN_ERR_CUDA, "cuTensorMapEncodeTiled(B) failed with code " + std::to_string((int)r));
      return TFGNN_ERR_CUDA;
    }
  }
  const size_t smem_bytes = (size_t)stages * stage_bytes + (2 * stages + 2 * kFuMaxSlots) * sizeof(uint64_t) + 128 +
                            (size_t)gather_warps * q * row_bytes + 1024;
  TFGNN_REQUIRE(smem_bytes <= (size_t)kFuSmemLimit, "fused RGCN: shared memory budget exceeded");
  const int nv = (D + 127) / 128;
  // L2 set-aside for the evict_last (persisting) lines: the ring + the packed weights.  Without a carve-out
  // the evict_last hint is advisory only and the ring gets written back to HBM.
  {
    const int rc_l2 = ensure_l2_persist_carveout((size_t)grid * p.num_slots * tile_rows * D * sizeof(float) +
                                                 (size_t)2 * H * L * D * sizeof(float));
    if (rc_l2) return rc_l2;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(rows ? kRtThreads : kFuThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = split || rows ? 2u : 1u;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (rows) {
    const long long units = (p.m_tiles + 1) / 2;
    switch (nv) {
      case 1: TFGNN_CUDA(launch_fused_rows_nv<1>(cfg, map_a, map_b, p, units, grid / 2)); break;
      case 2: TFGNN_CUDA(launch_fused_rows_nv<2>(cfg, map_a, map_b, p, units, grid / 2)); break;
      case 3: TFGNN_CUDA(launch_fused_rows_nv<3>(cfg, map_a, map_b, p, units, grid / 2)); break;
      default: TFGNN_CUDA(launch_fused_rows_nv<4>(cfg, map_a, map_b, p, units, grid / 2)); break;
    }
    TFGNN_LAUNCH_CHECK();
    return 0;
  }
  switch (nv) {
    case 1: TFGNN_CUDA(launch_fused_nv<1>(cfg, map_a, map_b, p)); break;
    case 2: TFGNN_CUDA(launch_fused_nv<2>(cfg, map_a, map_b, p)); break;
    case 3: TFGNN_CUDA(launch_fused_nv<3>(cfg, map_a, map_b, p)); break;
    default: TFGNN_CUDA(launch_fused_nv<4>(cfg, map_a, map_b, p)); break;
  }
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn
