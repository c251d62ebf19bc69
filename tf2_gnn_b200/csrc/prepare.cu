// Per-batch preprocessing: edges sorted by (type, target) -> keyed CSR + in-degree table.
//
// Replaces calculate_type_to_num_incoming_edges (message_passing.py:230-263, recomputed by the
// reference every layer at :190) and the per-layer slicing of adjacency lists
// (message_passing.py:118-121,195-196) by one pass per batch.  All arithmetic is int32 and
// therefore bit-exact; the float32 in-degree table is an exact conversion (counts < 2^24).
#include "common.cuh"

namespace tfgnn {

// How an edge (src, tgt) enters the CSR: segment key and stored value.
enum CsrKind { kByTarget = 0, kBySource = 1, kBySourceOwned = 2 };
// kByTarget:      key tgt - off, value src          (kept when tgt - off < V)
// kBySource:      key src - off, value tgt          (TFGNN_PREPARE_TRANSPOSE: kept when src - off < V)
// kBySourceOwned: key src,       value tgt - off    (TFGNN_PREPARE_TRANSPOSE_OWNED: kept when tgt - off < V_own; V = V_src)
// Returns false for an edge this batch does not keep.  Both ids must already lie in [0, V_src).
__device__ __forceinline__ bool csr_entry(int2 st, int V, int off, int V_own, int kind, int* key, int* value) {
  if (kind == kBySourceOwned) {
    const unsigned t = (unsigned)(st.y - off);
    *key = st.x;
    *value = (int)t;
    return t < (unsigned)V_own;
  }
  if (kind == kBySource) { const int t0 = st.x; st.x = st.y; st.y = t0; }
  const unsigned t = (unsigned)(st.y - off);
  *key = (int)t;
  *value = st.x;
  return t < (unsigned)V;   // else: another shard's node
}

// ---- 1. histogram of edges per (type, key node) ------------------------------------------
__global__ void count_targets_kernel(PtrTable adj, CountTable E, int V, int V_src, int off, int V_own, int kind,
                                     int* __restrict__ counts, int* __restrict__ invalid) {
  const int l = blockIdx.y;
  const long long n = E.n[l];
  const int2* __restrict__ edges = reinterpret_cast<const int2*>(adj.p[l]);
  int bad = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int2 st = __ldg(edges + e);
    if ((unsigned)st.x < (unsigned)V_src && (unsigned)st.y < (unsigned)V_src) {
      int key, value;
      if (csr_entry(st, V, off, V_own, kind, &key, &value)) atomicAdd(counts + (long long)l * V + key, 1);
    } else {
      ++bad;
    }
  }
  if (bad) atomicAdd(invalid, bad);
}

// ---- 2. exclusive scan (three-phase, in place) ---------------------------------------------
constexpr int kScanThreads = 512;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ int block_exclusive_scan(int v, int* total_out) {
  __shared__ int warp_sums[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
    int wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    if (lane < kScanThreads / 32) warp_sums[lane] = wi - w;  // exclusive warp offsets
    if (lane == kScanThreads / 32 - 1) *total_out = wi;
  }
  __syncthreads();
  int res = incl - v + warp_sums[warp];
  __syncthreads();
  return res;
}

__global__ void scan_reduce_kernel(const int* __restrict__ data, long long n, int* __restrict__ block_sums) {
  __shared__ int total;
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  int s = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j)
    if (base + j < n) s += data[base + j];
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

__global__ void scan_block_sums_kernel(int* __restrict__ block_sums, int num_blocks) {
  __shared__ int total;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < num_blocks; base += kScanThreads) {
    int i = base + threadIdx.x;
    int v = i < num_blocks ? block_sums[i] : 0;
    int ex = block_exclusive_scan(v, &total);
    if (i < num_blocks) block_sums[i] = ex + carry;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
}

__global__ void scan_apply_kernel(int* __restrict__ data, long long n, const int* __restrict__ block_offsets) {
  __shared__ int total;
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  int v[kScanItems];
  int s = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    v[j] = base + j < n ? data[base + j] : 0;
    s += v[j];
  }
  int run = block_exclusive_scan(s, &total) + block_offsets[blockIdx.x];
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    if (base + j < n) data[base + j] = run;
    run += v[j];
  }
}

// ---- 3. fill: sources into their (type,target) segment -------------------------------------
__global__ void fill_sources_kernel(PtrTable adj, CountTable E, int V, int V_src, int off, int V_own, int kind,
                                    int* __restrict__ cursor, int* __restrict__ src_sorted) {
  const int l = blockIdx.y;
  const long long n = E.n[l];
  const int2* __restrict__ edges = reinterpret_cast<const int2*>(adj.p[l]);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int2 st = __ldg(edges + e);
    if ((unsigned)st.x < (unsigned)V_src && (unsigned)st.y < (unsigned)V_src) {
      int key, value;
      if (csr_entry(st, V, off, V_own, kind, &key, &value)) {
        int pos = atomicAdd(cursor + (long long)l * V + key, 1);
        src_sorted[pos] = value;
      }
    }
  }
}

// Canonical order inside every segment (ascending source id): the fill above lands edges in
// atomic-arrival order, which would make float sums differ from one prepare() to the next.
// Duplicate edges carry equal ids, so ascending order is a unique arrangement.
// One warp per segment; short segments (<=32) use a shuffle bitonic network, medium ones (<=256) an
// in-place odd-even transposition by the warp, hubs are queued for sort_long_segments_kernel.
__global__ void sort_segments_kernel(const int* __restrict__ row_ptr, long long num_segments,
                                     int* __restrict__ src_sorted, long long* __restrict__ long_list,
                                     int* __restrict__ long_count) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long num_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long s = warp_global; s < num_segments; s += num_warps) {
    const int beg = row_ptr[s], end = row_ptr[s + 1];
    const int len = end - beg;
    if (len <= 1) continue;
    if (len <= 32) {
      int v = lane < len ? src_sorted[beg + lane] : 0x7fffffff;
#pragma unroll
      for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
          int other = __shfl_xor_sync(0xffffffffu, v, j);
          bool up = ((lane & k) == 0);
          bool lower = ((lane & j) == 0);
          int mn = min(v, other), mx = max(v, other);
          v = (lower == up) ? mn : mx;
        }
      }
      if (lane < len) src_sorted[beg + lane] = v;
    } else if (len <= 256) {
      // odd-even transposition sort over global memory (L1/L2 resident), len phases.
      for (int phase = 0; phase < len; ++phase) {
        for (int i = (phase & 1) + 2 * lane; i + 1 < len; i += 64) {
          int a = src_sorted[beg + i], b = src_sorted[beg + i + 1];
          if (a > b) {
            src_sorted[beg + i] = b;
            src_sorted[beg + i + 1] = a;
          }
        }
        __syncwarp();
      }
    }
    else {
      // hubs: queued for the block-level sorter below
      if (lane == 0) {
        const int slot = atomicAdd(long_count, 1);
        long_list[slot] = s;
      }
    }
  }
}

// Hub segments (> 256 edges): in-place bitonic sort (all-ascending "flip + disperse" network, so the
// virtual +inf padding beyond the segment end never moves) by one CTA per segment over global memory
// (L2 resident).  Makes the summation order of every segment a function of the graph alone.
__global__ void __launch_bounds__(512) sort_long_segments_kernel(const int* __restrict__ row_ptr,
                                                                 const long long* __restrict__ long_list,
                                                                 const int* __restrict__ long_count,
                                                                 int* __restrict__ src_sorted) {
  const int count = *long_count;
  for (int li = blockIdx.x; li < count; li += gridDim.x) {
    const long long s = long_list[li];
    const int beg = row_ptr[s], n = row_ptr[s + 1] - beg;
    int* a = src_sorted + beg;
    int P = 1;
    while (P < n) P <<= 1;
    const int half = P >> 1;
    for (int k = 2; k <= P; k <<= 1) {
      const int hk = k >> 1;
      for (int i = threadIdx.x; i < half; i += blockDim.x) {  // flip: i-th pair mirrors inside its k-block
        const int blk = i / hk, off = i - blk * hk;
        const int lo = blk * k + off, hi = blk * k + k - 1 - off;
        if (hi < n) {
          const int x = a[lo], y = a[hi];
          if (x > y) { a[lo] = y; a[hi] = x; }
        }
      }
      __syncthreads();
      for (int j = k >> 2; j > 0; j >>= 1) {                   // disperse
        for (int i = threadIdx.x; i < half; i += blockDim.x) {
          const int blk = i / j, off = i - blk * j;
          const int lo = blk * 2 * j + off, hi = lo + j;
          if (hi < n) {
            const int x = a[lo], y = a[hi];
            if (x > y) { a[lo] = y; a[hi] = x; }
          }
        }
        __syncthreads();
      }
    }
  }
}

__global__ void in_degree_kernel(const int* __restrict__ row_ptr, long long num_segments,
                                 float* __restrict__ out) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < num_segments;
       s += (long long)gridDim.x * blockDim.x)
    out[s] = (float)(row_ptr[s + 1] - row_ptr[s]);
}

int exclusive_scan_inplace(int* data, long long n, int* block_sums_scratch, cudaStream_t st) {
  const int nb = ceil_div(n, kScanTile);
  scan_reduce_kernel<<<nb, kScanThreads, 0, st>>>(data, n, block_sums_scratch);
  TFGNN_LAUNCH_CHECK();
  scan_block_sums_kernel<<<1, kScanThreads, 0, st>>>(block_sums_scratch, nb);
  TFGNN_LAUNCH_CHECK();
  scan_apply_kernel<<<nb, kScanThreads, 0, st>>>(data, n, block_sums_scratch);
  TFGNN_LAUNCH_CHECK();
  return 0;
}

}  // namespace tfgnn

using namespace tfgnn;

static int prepare_impl(const int32_t* const* adj, const int64_t* num_edges, int32_t L, int64_t V_total,
                        int64_t tgt_begin, int64_t V, uint32_t prepare_flags, tfgnn_batch_t** out_batch,
                        void* stream) {
  TFGNN_REQUIRE(out_batch != nullptr, "out_batch is NULL");
  *out_batch = nullptr;
  TFGNN_REQUIRE(L >= 0 && L <= TFGNN_MAX_EDGE_TYPES, "num_edge_types must be in [0, 32]");
  TFGNN_REQUIRE(V_total >= 0 && V_total < (1ll << 31), "num_nodes must be in [0, 2^31)");
  TFGNN_REQUIRE(tgt_begin >= 0 && V >= 0 && tgt_begin + V <= V_total, "target range must lie inside [0, num_nodes]");
  TFGNN_REQUIRE(L == 0 || (adj != nullptr && num_edges != nullptr), "adj / num_edges is NULL");
  long long M = 0, maxE = 0;
  for (int l = 0; l < L; ++l) {
    TFGNN_REQUIRE(num_edges[l] >= 0, "negative edge count");
    TFGNN_REQUIRE(num_edges[l] == 0 || adj[l] != nullptr, "adjacency pointer is NULL");
    M += num_edges[l];
    maxE = num_edges[l] > maxE ? num_edges[l] : maxE;
  }
  const int kind = (prepare_flags & TFGNN_PREPARE_TRANSPOSE_OWNED) ? kBySourceOwned
                   : (prepare_flags & TFGNN_PREPARE_TRANSPOSE)    ? kBySource
                                                                  : kByTarget;
  const long long V_own = V;                 // edges kept: target (kBySourceOwned) or key node in [tgt_begin, +V)
  if (kind == kBySourceOwned) V = V_total;   // segments per type: every global source
  const long long S = (long long)L * V;  // number of segments
  TFGNN_REQUIRE(M < (1ll << 31) - 1 && S < (1ll << 31) - 1,
                "batch too large for int32 CSR (shard it across GPUs)");
  cudaStream_t st = (cudaStream_t)stream;

  tfgnn_batch* b = new tfgnn_batch();
  b->V = V;
  b->V_src = V_total;
  b->tgt_off = kind == kBySourceOwned ? 0 : tgt_begin;
  b->owned_transpose = kind == kBySourceOwned;
  b->own_begin = tgt_begin;
  b->own_count = V_own;
  b->L = L;
  b->M_in = M;
  int rc = 0;
  auto fail = [&](int code) {
    tfgnn_b200_free_batch(b);
    return code;
  };
#define TRY(expr)                      \
  do {                                 \
    rc = (expr);                       \
    if (rc) return fail(rc);           \
  } while (0)
#define TRY_CUDA(expr) TRY(check_cuda((expr), #expr, __FILE__, __LINE__))

  TRY_CUDA(cudaGetDevice(&b->device));
  TRY(batch_enter(b, st));
  TRY(pool_alloc((void**)&b->row_ptr, (size_t)(S + 1) * sizeof(int), st));
  TRY(pool_alloc((void**)&b->src_sorted, (size_t)(M > 0 ? M : 1) * sizeof(int), st));
  TRY(pool_alloc((void**)&b->invalid_count, sizeof(int), st));
  TRY_CUDA(cudaMemsetAsync(b->row_ptr, 0, (size_t)(S + 1) * sizeof(int), st));
  TRY_CUDA(cudaMemsetAsync(b->invalid_count, 0, sizeof(int), st));

  PtrTable pt{};
  CountTable ct{};
  for (int l = 0; l < L; ++l) {
    pt.p[l] = adj[l];
    ct.n[l] = num_edges[l];
    b->adj[l] = adj[l];
    b->E[l] = num_edges[l];
  }
  if (M > 0 && V > 0) {
    int bx = ceil_div(maxE, 256);
    if (bx > 132 * 16) bx = 132 * 16;
    if (bx < 1) bx = 1;
    dim3 grid(bx, L);
    count_targets_kernel<<<grid, 256, 0, st>>>(pt, ct, (int)V, (int)V_total, (int)tgt_begin, (int)V_own, kind,
                                               b->row_ptr, b->invalid_count);
    g_launch_count.fetch_add(1);
    TRY_CUDA(cudaGetLastError());
  }
  // scan of the counts, then the sources in segment order.  The block sums, the fill cursor and the hub list belong to this
  // call alone: they are freed on `st` when the lambda returns, before fail() can free the batch.
  auto scan_and_fill = [&]() -> int {
    PoolBuffer bs{st};
    int r = bs.alloc((size_t)ceil_div(S + 1, kScanTile) * sizeof(int));
    if (!r) r = exclusive_scan_inplace(b->row_ptr, S + 1, (int*)bs.p, st);
    if (r || M == 0 || V == 0) return r;
    PoolBuffer cursor{st};
    r = cursor.alloc((size_t)(S + 1) * sizeof(int));
    if (r) return r;
    TFGNN_CUDA(cudaMemcpyAsync(cursor.p, b->row_ptr, (size_t)S * sizeof(int), cudaMemcpyDeviceToDevice, st));
    int bx = ceil_div(maxE, 256);
    if (bx > 132 * 16) bx = 132 * 16;
    dim3 grid(bx, L);
    fill_sources_kernel<<<grid, 256, 0, st>>>(pt, ct, (int)V, (int)V_total, (int)tgt_begin, (int)V_own, kind,
                                              (int*)cursor.p, b->src_sorted);
    g_launch_count.fetch_add(1);
    TFGNN_CUDA(cudaGetLastError());
    long long warps_needed = S;
    int blocks = ceil_div(warps_needed * 32, 256);
    if (blocks > 132 * 32) blocks = 132 * 32;
    // a segment longer than 256 edges is a "hub"; there are at most M/257 of them
    const long long max_long = M / 257 + 1;
    PoolBuffer long_buf{st};
    r = long_buf.alloc((size_t)max_long * sizeof(long long) + 16);
    if (r) return r;
    int* long_count = reinterpret_cast<int*>(long_buf.p);
    long long* long_list = reinterpret_cast<long long*>(reinterpret_cast<char*>(long_buf.p) + 16);
    TFGNN_CUDA(cudaMemsetAsync(long_count, 0, sizeof(int), st));
    sort_segments_kernel<<<blocks, 256, 0, st>>>(b->row_ptr, S, b->src_sorted, long_list, long_count);
    g_launch_count.fetch_add(1);
    TFGNN_CUDA(cudaGetLastError());
    sort_long_segments_kernel<<<132 * 2, 512, 0, st>>>(b->row_ptr, long_list, long_count, b->src_sorted);
    g_launch_count.fetch_add(1);
    TFGNN_CUDA(cudaGetLastError());
    return 0;
  };
  TRY(scan_and_fill());
  if (prepare_flags & TFGNN_PREPARE_VALIDATE) {
    int bad = 0;
    TRY_CUDA(cudaMemcpyAsync(&bad, b->invalid_count, sizeof(int), cudaMemcpyDeviceToHost, st));
    TRY_CUDA(cudaStreamSynchronize(st));
    if (bad) {
      set_error(TFGNN_ERR_INDEX_OUT_OF_RANGE,
                std::to_string(bad) + " edge(s) reference a node outside [0, " + std::to_string(V_total) + ")");
      return fail(TFGNN_ERR_INDEX_OUT_OF_RANGE);
    }
  }
#undef TRY
#undef TRY_CUDA
  *out_batch = b;
  return 0;
}

extern "C" int tfgnn_b200_prepare(const int32_t* const* adj, const int64_t* num_edges, int32_t L, int64_t V,
                                  uint32_t prepare_flags, tfgnn_batch_t** out_batch, void* stream) {
  return prepare_impl(adj, num_edges, L, V, 0, V, prepare_flags, out_batch, stream);
}

extern "C" int tfgnn_b200_prepare_sharded(const int32_t* const* adj, const int64_t* num_edges, int32_t L,
                                          int64_t num_nodes_total, int64_t target_begin, int64_t target_count,
                                          uint32_t prepare_flags, tfgnn_batch_t** out_batch, void* stream) {
  return prepare_impl(adj, num_edges, L, num_nodes_total, target_begin, target_count, prepare_flags, out_batch,
                      stream);
}

extern "C" int tfgnn_b200_free_batch(tfgnn_batch_t* b) {
  if (!b) return 0;
  // stream-ordered frees behind the last work enqueued for this batch: no device synchronisation
  pool_free(b->row_ptr, b->cur_stream);
  pool_free(b->src_sorted, b->cur_stream);
  pool_free(b->invalid_count, b->cur_stream);
  if (b->ev_switch) cudaEventDestroy(b->ev_switch);
  if (b->pipe_ready) {
    cudaStreamDestroy(b->pipe_gather);
    cudaStreamDestroy(b->pipe_gemm);
    cudaEventDestroy(b->ev_fork);
    cudaEventDestroy(b->ev_join_g);
    cudaEventDestroy(b->ev_join_m);
    for (int i = 0; i < tfgnn_batch::kPipeBufs; ++i) {
      cudaEventDestroy(b->ev_g[i]);
      cudaEventDestroy(b->ev_m[i]);
    }
  }
  delete b;
  return 0;
}

extern "C" int tfgnn_b200_batch_info(const tfgnn_batch_t* b, int64_t* V, int32_t* L, int64_t* M,
                                     const int32_t** row_ptr, const int32_t** src_sorted) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  if (V) *V = b->V;
  if (L) *L = b->L;
  if (M) *M = b->M_in;
  if (row_ptr) *row_ptr = b->row_ptr;
  if (src_sorted) *src_sorted = b->src_sorted;
  return 0;
}

extern "C" int tfgnn_b200_batch_export_csr(const tfgnn_batch_t* b, int32_t* row_ptr_out, int32_t* src_sorted_out,
                                           void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  // a read of the CSR enters the batch like a layer call: it waits for the prepare on another stream, and the free
  // (on the last stream entered) waits for it.  The stream fields are bookkeeping, not the batch's contents.
  const int rc = batch_enter(const_cast<tfgnn_batch*>(b), st);
  if (rc) return rc;
  const long long S = (long long)b->L * b->V;
  if (row_ptr_out)
    TFGNN_CUDA(cudaMemcpyAsync(row_ptr_out, b->row_ptr, (size_t)(S + 1) * sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (src_sorted_out && b->M_in > 0)
    TFGNN_CUDA(cudaMemcpyAsync(src_sorted_out, b->src_sorted, (size_t)b->M_in * sizeof(int), cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int tfgnn_b200_in_degree(const tfgnn_batch_t* b, float* out, void* stream) {
  TFGNN_REQUIRE(b != nullptr, "batch is NULL");
  const long long S = (long long)b->L * b->V;
  if (S == 0) return 0;
  TFGNN_REQUIRE(out != nullptr, "out is NULL");
  const int rc = batch_enter(const_cast<tfgnn_batch*>(b), (cudaStream_t)stream);   // as in tfgnn_b200_batch_export_csr
  if (rc) return rc;
  int blocks = ceil_div(S, 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  in_degree_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(b->row_ptr, S, out);
  TFGNN_LAUNCH_CHECK();
  return 0;
}
