// On-device batch builder (SURVEY.md §8f-2): the integer bookkeeping that shapes what the message-passing path
// consumes, moved off the host's Python loops.  HBM-bound int32 copies; everything is bit-exact by construction.
//
//   tfgnn_b200_process_adjacency   tf2_gnn/data/utils.py:9-58   backward edges (tied into the forward type or as fresh
//                                  types), self-loop type at a chosen slot, in-degree table [L, V]
//   tfgnn_b200_assemble_batch      tf2_gnn/data/graph_dataset.py:161-246   disjoint union of graphs: node ids offset by the
//                                  running node count, node_to_graph_map = constant block per graph
//
// The dataset lives packed on the device (all graphs of an edge type back to back, graph-local ids, int64 offset
// tables); a minibatch is a list of graph ids.  One scan kernel turns the ids into batch offsets, one fill kernel per
// output array does a binary search over <= ~1e5 graph offsets per element (L1/L2-resident) and one 8-byte copy.
#include "common.cuh"

namespace tfgnn {

constexpr int MAX_TYPES_PLUS_ONE = TFGNN_MAX_EDGE_TYPES + 1;

static int bb_grid(long long n) {
  long long g = (n + 255) / 256;
  return (int)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}

// ---- process_adjacency_lists -------------------------------------------------------------------------------
// dst[e] = flip ? (src[e].tgt, src[e].src) : src[e]
__global__ void copy_pairs_kernel(const int2* __restrict__ src, long long n, int flip, int2* __restrict__ dst) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int2 p = src[i];
    dst[i] = flip ? make_int2(p.y, p.x) : p;
  }
}
__global__ void iota_pairs_kernel(long long n, int2* __restrict__ dst) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = make_int2((int)i, (int)i);
}
// counts[tgt] += 1 (int32; exact, order-independent)
__global__ void count_in_kernel(const int2* __restrict__ adj, long long n, long long V, int* __restrict__ counts) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = adj[i].y;
    if ((unsigned long long)(long long)t < (unsigned long long)V) atomicAdd(counts + t, 1);
  }
}
__global__ void int_to_float_inplace_kernel(float* __restrict__ buf, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    buf[i] = (float)reinterpret_cast<const int*>(buf)[i];
}

// ---- assemble_batch ------------------------------------------------------------------------------------------
// Block b scans one count table over the batch's graphs: b = 0 node counts, b >= 1 edge counts of type b-1.
// ws[b * (Gb + 1) + g] = exclusive prefix, ws[b * (Gb + 1) + Gb] = total.
struct OffsetTables {
  const long long* t[MAX_TYPES_PLUS_ONE];   // [0] node_offsets, [1 + t] edge_offsets of type t; each int64[G + 1]
};
__global__ void batch_scan_kernel(OffsetTables tabs, const int* __restrict__ graph_ids, int Gb, long long G,
                                  long long* __restrict__ ws) {
  __shared__ long long warp_sums[32];
  __shared__ long long carry_s;
  const long long* off = tabs.t[blockIdx.x];
  long long* out = ws + (long long)blockIdx.x * (Gb + 1);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < Gb; base += blockDim.x) {
    const int g = base + threadIdx.x;
    long long c = 0;
    if (g < Gb) {
      const long long id = graph_ids[g];
      if (id >= 0 && id < G) c = off[id + 1] - off[id];
    }
    long long x = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      long long s = lane < nwarps ? warp_sums[lane] : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, s, d);
        if (lane >= d) s += y;
      }
      warp_sums[lane] = s;   // inclusive over warps
    }
    __syncthreads();
    const long long carry = carry_s;
    const long long before = carry + (warp ? warp_sums[warp - 1] : 0) + (x - c);
    if (g < Gb) out[g] = before;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry_s = carry + warp_sums[nwarps - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[Gb] = carry_s;
}

// largest g in [0, Gb) with off[g] <= i  (off non-decreasing, off[0] = 0, i < off[Gb])
__device__ __forceinline__ int find_graph(const long long* __restrict__ off, int Gb, long long i) {
  int lo = 0, hi = Gb;   // invariant: off[lo] <= i < off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// node_to_graph_map[v] = g (batch-local index, graph_dataset.py:211-217); src_row[v] = the node's row in the packed store.
// v counts from batch row v0: a row window [v0, v0 + Vb) of the batch (v0 = 0 for the whole batch).
__global__ void fill_nodes_kernel(const long long* __restrict__ node_off_batch, int Gb,
                                  const long long* __restrict__ node_offsets, const int* __restrict__ graph_ids,
                                  long long v0, long long Vb, int* __restrict__ node_to_graph_map, int* __restrict__ src_row) {
  const long long total = node_off_batch[Gb];   // a caller-supplied size larger than the real batch is not followed
  if (Vb > total - v0) Vb = total - v0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < Vb; i += (long long)gridDim.x * blockDim.x) {
    const long long v = v0 + i;
    const int g = find_graph(node_off_batch, Gb, v);
    if (node_to_graph_map) node_to_graph_map[i] = g;
    if (src_row) src_row[i] = (int)(node_offsets[graph_ids[g]] + (v - node_off_batch[g]));
  }
}

// adjacency_list_t[e] = stored pair + running node count of its graph (graph_dataset.py:218-222).  With row_end >= 0 only
// the edges of the graphs that overlap batch rows [row_begin, row_end) are written, from out[0] on and in batch order:
// the sub-range [edge_off_batch[g_first], edge_off_batch[g_last + 1]) of the whole batch's list.
__global__ void fill_edges_kernel(const long long* __restrict__ edge_off_batch, const long long* __restrict__ node_off_batch,
                                  int Gb, const long long* __restrict__ edge_offsets, const int* __restrict__ graph_ids,
                                  const int2* __restrict__ edges, long long row_begin, long long row_end, long long Eb,
                                  int2* __restrict__ out) {
  long long e0 = 0, e1 = edge_off_batch[Gb];
  if (row_end >= 0) {
    if (row_end > node_off_batch[Gb]) row_end = node_off_batch[Gb];
    e0 = e1 = 0;
    if (row_begin < row_end) {
      e0 = edge_off_batch[find_graph(node_off_batch, Gb, row_begin)];
      e1 = edge_off_batch[find_graph(node_off_batch, Gb, row_end - 1) + 1];
    }
  }
  if (Eb > e1 - e0) Eb = e1 - e0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < Eb; i += (long long)gridDim.x * blockDim.x) {
    const long long e = e0 + i;
    const int g = find_graph(edge_off_batch, Gb, e);
    const long long src_e = edge_offsets[graph_ids[g]] + (e - edge_off_batch[g]);
    const int shift = (int)node_off_batch[g];
    const int2 p = edges[src_e];
    out[i] = make_int2(p.x + shift, p.y + shift);
  }
}

// The launches of assemble_batch over batch rows [row_begin, row_end); row_end < 0: the whole batch.  Arguments checked.
static int assemble_launch(const int64_t* node_offsets, const int64_t* const* edge_offsets, const int32_t* const* edges,
                           int num_edge_types, int64_t num_graphs_total, const int32_t* graph_ids, int Gb,
                           long long row_begin, long long row_end, long long num_rows, const int64_t* num_edges,
                           int32_t* node_to_graph_map, int32_t* node_source_rows, int32_t* const* adjacency_lists,
                           void* workspace, cudaStream_t st) {
  OffsetTables tabs{};
  tabs.t[0] = reinterpret_cast<const long long*>(node_offsets);
  for (int t = 0; t < num_edge_types; ++t) {
    TFGNN_REQUIRE(edge_offsets[t] != nullptr, "NULL edge offset table");
    tabs.t[1 + t] = reinterpret_cast<const long long*>(edge_offsets[t]);
  }
  long long* ws = reinterpret_cast<long long*>(workspace);
  batch_scan_kernel<<<num_edge_types + 1, 1024, 0, st>>>(tabs, graph_ids, Gb, num_graphs_total, ws);
  TFGNN_LAUNCH_CHECK();
  if (num_rows > 0 && (node_to_graph_map || node_source_rows)) {
    fill_nodes_kernel<<<bb_grid(num_rows), 256, 0, st>>>(ws, Gb, reinterpret_cast<const long long*>(node_offsets),
                                                       graph_ids, row_begin, num_rows, node_to_graph_map,
                                                       node_source_rows);
    TFGNN_LAUNCH_CHECK();
  }
  for (int t = 0; t < num_edge_types; ++t) {
    const long long Eb = num_edges[t];
    TFGNN_REQUIRE(Eb >= 0, "negative edge count");
    if (Eb == 0) continue;
    TFGNN_REQUIRE(edges[t] && adjacency_lists[t], "NULL edge list");
    fill_edges_kernel<<<bb_grid(Eb), 256, 0, st>>>(ws + (size_t)(1 + t) * (Gb + 1), ws, Gb,
                                                 reinterpret_cast<const long long*>(edge_offsets[t]), graph_ids,
                                                 reinterpret_cast<const int2*>(edges[t]), row_begin, row_end, Eb,
                                                 reinterpret_cast<int2*>(adjacency_lists[t]));
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace tfgnn

using namespace tfgnn;

// Layout of the processed adjacency lists, exactly as data/utils.py:91-113 builds it: slot -> (forward type, role).
//   role 0: forward edges only, 1: forward then flipped (tied), 2: flipped only (fresh backward type), 3: self loops
struct AdjSlot { int type; int role; };
static int plan_slots(int T, const int32_t* tied, int add_self_loops, int self_loop_type, AdjSlot* slots, int* L_out) {
  int n = 0;
  for (int t = 0; t < T; ++t) slots[n++] = {t, tied && tied[t] ? 1 : 0};
  for (int t = 0; t < T; ++t)
    if (!(tied && tied[t])) slots[n++] = {t, 2};
  if (add_self_loops) {
    if (self_loop_type < -(n + 1) || self_loop_type > n) return -1;   // list.insert range accepted by the reference's assert
    const int slot = self_loop_type < 0 ? self_loop_type + n + 1 : self_loop_type;
    for (int i = n; i > slot; --i) slots[i] = slots[i - 1];
    slots[slot] = {-1, 3};
    ++n;
  }
  *L_out = n;
  return 0;
}

extern "C" int tfgnn_b200_process_adjacency_sizes(const int64_t* num_edges_fwd, int32_t num_fwd_types, int64_t num_nodes,
                                                  int32_t add_self_loop_edges, const int32_t* tied,
                                                  int32_t self_loop_edge_type, int64_t* num_edges_out,
                                                  int32_t* num_types_out) {
  TFGNN_REQUIRE(num_fwd_types >= 0 && 2 * num_fwd_types + 1 <= TFGNN_MAX_EDGE_TYPES, "too many edge types");
  TFGNN_REQUIRE(num_nodes >= 0 && num_types_out != nullptr, "bad process_adjacency arguments");
  TFGNN_REQUIRE(num_fwd_types == 0 || num_edges_fwd != nullptr, "num_edges_fwd is NULL");
  AdjSlot slots[TFGNN_MAX_EDGE_TYPES + 1];
  int L = 0;
  TFGNN_REQUIRE(plan_slots(num_fwd_types, tied, add_self_loop_edges, self_loop_edge_type, slots, &L) == 0,
                "self_loop_edge_type out of range");
  *num_types_out = L;
  if (num_edges_out)
    for (int l = 0; l < L; ++l) {
      const AdjSlot s = slots[l];
      num_edges_out[l] = s.role == 3 ? num_nodes : num_edges_fwd[s.type] * (s.role == 1 ? 2 : 1);
    }
  return 0;
}

extern "C" int tfgnn_b200_process_adjacency(const int32_t* const* adjacency_fwd, const int64_t* num_edges_fwd,
                                            int32_t num_fwd_types, int64_t num_nodes, int32_t add_self_loop_edges,
                                            const int32_t* tied, int32_t self_loop_edge_type,
                                            int32_t* const* adjacency_out, int32_t num_types_out,
                                            float* type_to_num_incoming_edges, void* stream) {
  TFGNN_REQUIRE(num_fwd_types >= 0 && 2 * num_fwd_types + 1 <= TFGNN_MAX_EDGE_TYPES, "too many edge types");
  TFGNN_REQUIRE(num_nodes >= 0 && num_nodes < (1ll << 31), "num_nodes out of range");
  cudaStream_t st = (cudaStream_t)stream;
  AdjSlot slots[TFGNN_MAX_EDGE_TYPES + 1];
  int L = 0;
  TFGNN_REQUIRE(plan_slots(num_fwd_types, tied, add_self_loop_edges, self_loop_edge_type, slots, &L) == 0,
                "self_loop_edge_type out of range");
  TFGNN_REQUIRE(L == num_types_out, "num_types_out does not match the processed layout (call tfgnn_b200_process_adjacency_sizes)");
  TFGNN_REQUIRE(L == 0 || adjacency_out != nullptr, "adjacency_out is NULL");
  if (type_to_num_incoming_edges && L > 0 && num_nodes > 0)
    TFGNN_CUDA(cudaMemsetAsync(type_to_num_incoming_edges, 0, (size_t)L * num_nodes * sizeof(float), st));
  for (int l = 0; l < L; ++l) {
    const AdjSlot s = slots[l];
    int2* dst = reinterpret_cast<int2*>(adjacency_out[l]);
    long long n_out = 0;
    if (s.role == 3) {
      n_out = num_nodes;
      if (n_out > 0) {
        TFGNN_REQUIRE(dst != nullptr, "NULL output list");
        iota_pairs_kernel<<<bb_grid(n_out), 256, 0, st>>>(n_out, dst);
        TFGNN_LAUNCH_CHECK();
      }
    } else {
      const long long n = num_edges_fwd[s.type];
      TFGNN_REQUIRE(n >= 0, "negative edge count");
      const int2* src = reinterpret_cast<const int2*>(adjacency_fwd[s.type]);
      n_out = n * (s.role == 1 ? 2 : 1);
      if (n > 0) {
        TFGNN_REQUIRE(src != nullptr && dst != nullptr, "NULL adjacency list");
        if (s.role != 2) {
          copy_pairs_kernel<<<bb_grid(n), 256, 0, st>>>(src, n, 0, dst);
          TFGNN_LAUNCH_CHECK();
        }
        if (s.role != 0) {
          copy_pairs_kernel<<<bb_grid(n), 256, 0, st>>>(src, n, 1, dst + (s.role == 1 ? n : 0));
          TFGNN_LAUNCH_CHECK();
        }
      }
    }
    if (type_to_num_incoming_edges && n_out > 0 && num_nodes > 0) {
      count_in_kernel<<<bb_grid(n_out), 256, 0, st>>>(dst, n_out, num_nodes,
                                                     reinterpret_cast<int*>(type_to_num_incoming_edges) + (size_t)l * num_nodes);
      TFGNN_LAUNCH_CHECK();
    }
  }
  if (type_to_num_incoming_edges && L > 0 && num_nodes > 0) {
    int_to_float_inplace_kernel<<<bb_grid((long long)L * num_nodes), 256, 0, st>>>(type_to_num_incoming_edges,
                                                                                  (long long)L * num_nodes);
    TFGNN_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" size_t tfgnn_b200_assemble_batch_workspace_bytes(int32_t num_edge_types, int32_t num_graphs_in_batch) {
  return (size_t)(num_edge_types + 1) * ((size_t)num_graphs_in_batch + 1) * sizeof(long long);
}

extern "C" int tfgnn_b200_assemble_batch(const int64_t* node_offsets, const int64_t* const* edge_offsets,
                                         const int32_t* const* edges, int32_t num_edge_types, int64_t num_graphs_total,
                                         const int32_t* graph_ids, int32_t num_graphs_in_batch,
                                         int64_t num_nodes_in_batch, const int64_t* num_edges_in_batch,
                                         int32_t* node_to_graph_map, int32_t* node_source_rows,
                                         int32_t* const* adjacency_lists, void* workspace, void* stream) {
  TFGNN_REQUIRE(num_edge_types >= 0 && num_edge_types <= TFGNN_MAX_EDGE_TYPES, "too many edge types");
  TFGNN_REQUIRE(num_graphs_in_batch >= 0 && num_graphs_total >= 0 && num_nodes_in_batch >= 0, "negative size");
  TFGNN_REQUIRE(num_nodes_in_batch < (1ll << 31), "batch has too many nodes for int32 ids");
  if (num_graphs_in_batch == 0) return 0;
  TFGNN_REQUIRE(node_offsets && graph_ids && workspace, "NULL pointer");
  TFGNN_REQUIRE(num_edge_types == 0 || (edge_offsets && edges && adjacency_lists && num_edges_in_batch), "NULL edge tables");
  return assemble_launch(node_offsets, edge_offsets, edges, num_edge_types, num_graphs_total, graph_ids,
                         num_graphs_in_batch, 0, -1, num_nodes_in_batch, num_edges_in_batch, node_to_graph_map,
                         node_source_rows, adjacency_lists, workspace, (cudaStream_t)stream);
}

extern "C" int tfgnn_b200_assemble_batch_rows(const int64_t* node_offsets, const int64_t* const* edge_offsets,
                                              const int32_t* const* edges, int32_t num_edge_types, int64_t num_graphs_total,
                                              const int32_t* graph_ids, int32_t num_graphs_in_batch,
                                              int64_t num_nodes_in_batch, const int64_t* num_edges_in_window,
                                              int64_t row_begin, int64_t row_count, int32_t* node_to_graph_map,
                                              int32_t* node_source_rows, int32_t* const* adjacency_lists, void* workspace,
                                              void* stream) {
  TFGNN_REQUIRE(num_edge_types >= 0 && num_edge_types <= TFGNN_MAX_EDGE_TYPES,
                "tfgnn_b200_assemble_batch_rows: too many edge types");
  TFGNN_REQUIRE(num_graphs_in_batch >= 0 && num_graphs_total >= 0 && num_nodes_in_batch >= 0,
                "tfgnn_b200_assemble_batch_rows: negative size");
  TFGNN_REQUIRE(num_nodes_in_batch < (1ll << 31), "tfgnn_b200_assemble_batch_rows: batch has too many nodes for int32 ids");
  TFGNN_REQUIRE(row_begin >= 0 && row_count >= 0 && row_begin + row_count <= num_nodes_in_batch,
                "tfgnn_b200_assemble_batch_rows: row window outside the batch");
  if (num_graphs_in_batch == 0 || row_count == 0) return 0;
  TFGNN_REQUIRE(node_offsets && graph_ids && workspace, "tfgnn_b200_assemble_batch_rows: NULL pointer");
  TFGNN_REQUIRE(num_edge_types == 0 || (edge_offsets && edges && adjacency_lists && num_edges_in_window),
                "tfgnn_b200_assemble_batch_rows: NULL edge tables");
  return assemble_launch(node_offsets, edge_offsets, edges, num_edge_types, num_graphs_total, graph_ids,
                         num_graphs_in_batch, row_begin, row_begin + row_count, row_count, num_edges_in_window,
                         node_to_graph_map, node_source_rows, adjacency_lists, workspace, (cudaStream_t)stream);
}
