// One consumer warpgroup's share of a 128-row output tile on the sm_90a tensor cores, with fp32-level accuracy ("3xTF32"):
//     x = x_hi + x_lo (tf32 split),   A*B ~= A_hi*B_hi + (A_lo*B_hi + A_hi*B_lo)     (dropped term ~2^-22 relative)
// The warpgroup owns rows [64 wg, 64 wg + 64) of the tile and keeps two fp32 accumulators in registers: the main product and
// the two small correction products, which are added only in the epilogue (the tensor core adds each K step into its
// accumulator with truncation; keeping the small terms apart keeps that bias off the large-magnitude sum).
// Used by the node-level GEMM (gemm_tc.cu) and the fused RGCN layer (fused_rgcn.cu).
#pragma once
#include "sm90_ptx.cuh"
#include "wgmma_ops.cuh"

namespace tfgnn {

template <int BN>
struct HalfTileAcc {
  float main[BN / 2];
  float corr[BN / 2];
};

// Splits this warpgroup's 64 rows of the raw fp32 A tile (128 rows of ROW_BYTES at a_tile, TMA-swizzled) in place: the
// tile becomes tf32(a), and the tile at a_tile + 128 * ROW_BYTES the correction operand - tf32(a - tf32(a)), or with
// corr_bf16 the bf16 pair (a | a - tf32(a)) (sm90_ptx.cuh).  Position-preserving, so independent of the swizzle.
template <int ROW_BYTES>
__device__ __forceinline__ void split_a_half(uint32_t a_tile, int wg, int t, int corr_bf16) {
  const uint32_t a_s = a_tile + (uint32_t)(wg * 64 * ROW_BYTES) + (uint32_t)t * 16u;
  const uint32_t lo_s = a_s + 128u * ROW_BYTES;
  constexpr int kIt = 64 * ROW_BYTES / 16 / 128;
  float4 xs[kIt];
#pragma unroll
  for (int i = 0; i < kIt; ++i) xs[i] = ptx::lds_f4(a_s + (uint32_t)i * 2048u);
#pragma unroll
  for (int i = 0; i < kIt; ++i) {
    const float4 x = xs[i];
    float4 h;
    h.x = ptx::tf32_hi(x.x); h.y = ptx::tf32_hi(x.y); h.z = ptx::tf32_hi(x.z); h.w = ptx::tf32_hi(x.w);
    ptx::sts_f4(a_s + (uint32_t)i * 2048u, h);
    if (corr_bf16) {
      uint4 w;
      w.x = ptx::pack_bf16x2(x.x - h.x, x.x); w.y = ptx::pack_bf16x2(x.y - h.y, x.y);
      w.z = ptx::pack_bf16x2(x.z - h.z, x.z); w.w = ptx::pack_bf16x2(x.w - h.w, x.w);
      ptx::sts_u4(lo_s + (uint32_t)i * 2048u, w);
    } else {
      float4 l;
      l.x = ptx::tf32_hi(x.x - h.x); l.y = ptx::tf32_hi(x.y - h.y);
      l.z = ptx::tf32_hi(x.z - h.z); l.w = ptx::tf32_hi(x.w - h.w);
      ptx::sts_f4(lo_s + (uint32_t)i * 2048u, l);
    }
  }
}

// Issues (does not wait for) the MMAs of one K block of ROW_BYTES / 4 floats: B is the pre-split weight tile (BN rows of
// tf32 hi at b_tile, BN rows of the correction operand right after it).  first: the block starts the tile's accumulation.
template <int BN, int ROW_BYTES>
__device__ __forceinline__ void mma_kblock(HalfTileAcc<BN>& c, uint32_t a_tile, uint32_t b_tile, int wg, int corr_bf16,
                                           bool first) {
  const uint32_t a_hi = a_tile + (uint32_t)(wg * 64 * ROW_BYTES);
  const uint64_t da_hi = ptx::gmma_desc_k<ROW_BYTES>(a_hi);
  const uint64_t da_lo = ptx::gmma_desc_k<ROW_BYTES>(a_hi + 128u * ROW_BYTES);
  const uint64_t db_hi = ptx::gmma_desc_k<ROW_BYTES>(b_tile);
  const uint64_t db_lo = ptx::gmma_desc_k<ROW_BYTES>(b_tile + (uint32_t)(BN * ROW_BYTES));
#pragma unroll
  for (int k = 0; k < ROW_BYTES / 32; ++k) {
    const uint64_t adv = (uint64_t)(k * 32 >> 4);   // 8 tf32 (or 16 bf16) = 32 B along K inside the swizzle row
    const int acc = (first && k == 0) ? 0 : 1;
    if (corr_bf16) {
      ptx::wgmma_bf16<BN>(c.corr, da_lo + adv, db_lo + adv, acc);   // pair tiles: a lo(b) + lo(a) b
    } else {
      ptx::wgmma_tf32<BN>(c.corr, da_lo + adv, db_hi + adv, acc);
      ptx::wgmma_tf32<BN>(c.corr, da_hi + adv, db_lo + adv, 1);
    }
    ptx::wgmma_tf32<BN>(c.main, da_hi + adv, db_hi + adv, acc);
  }
}

// After wgmma_wait<0>: pins the accumulators so no access is moved above the wait.
template <int BN>
__device__ __forceinline__ void fence_acc(HalfTileAcc<BN>& c) {
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) {
    ptx::reg_fence(c.main[j]);
    ptx::reg_fence(c.corr[j]);
  }
}

// Row `h` (0: row 16 w + lane / 4, 1: that row + 8) of this thread's accumulator fragment, main + correction, in column order:
// v[2 i + e] is tile column 8 i + 2 (lane % 4) + e.
template <int BN>
__device__ __forceinline__ void acc_row(const HalfTileAcc<BN>& c, int h, float (&v)[BN / 4]) {
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    v[2 * i] = c.main[4 * i + 2 * h] + c.corr[4 * i + 2 * h];
    v[2 * i + 1] = c.main[4 * i + 2 * h + 1] + c.corr[4 * i + 2 * h + 1];
  }
}

}  // namespace tfgnn
