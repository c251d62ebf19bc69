// Shared helpers for the tfgnn_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include <string>

#include "../../include/tfgnn_b200.h"

namespace tfgnn {

constexpr float kSmallNumber = 1e-7f;       // tf2_gnn/utils/constants.py:2
constexpr float kLeakyReluAlpha = 0.2f;     // tf.nn.leaky_relu default
constexpr float kSeluAlpha = 1.6732632423543772f;
constexpr float kSeluScale = 1.0507009873554805f;
constexpr float kLowestFloat = -3.402823466e+38f;  // tf.math.unsorted_segment_max identity

extern std::atomic<long long> g_launch_count;
void set_error(int code, const std::string& msg);
int last_error_code();

// Returns 0 or sets the thread-local error and returns TFGNN_ERR_CUDA.
int check_cuda(cudaError_t e, const char* what, const char* file, int line);
#define TFGNN_CUDA(expr)                                                        \
  do {                                                                          \
    int _rc = ::tfgnn::check_cuda((expr), #expr, __FILE__, __LINE__);           \
    if (_rc) return _rc;                                                        \
  } while (0)
#define TFGNN_LAUNCH_CHECK()                                                    \
  do {                                                                          \
    ::tfgnn::g_launch_count.fetch_add(1, std::memory_order_relaxed);            \
    TFGNN_CUDA(cudaGetLastError());                                             \
  } while (0)
#define TFGNN_REQUIRE(cond, msg)                                                \
  do {                                                                          \
    if (!(cond)) {                                                              \
      ::tfgnn::set_error(TFGNN_ERR_INVALID_ARGUMENT, std::string(msg));         \
      return TFGNN_ERR_INVALID_ARGUMENT;                                        \
    }                                                                           \
  } while (0)

// Activation table (tf2_gnn/utils/param_helpers.py:22-42).  tanhf/expm1f are the accurate
// libdevice versions: parity target is 1e-5 relative to the fp32 reference.
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case TFGNN_ACT_RELU: return fmaxf(x, 0.0f);
    case TFGNN_ACT_TANH: return tanhf(x);
    case TFGNN_ACT_LEAKY_RELU: return x > 0.0f ? x : kLeakyReluAlpha * x;
    case TFGNN_ACT_ELU: return x > 0.0f ? x : expm1f(x);
    case TFGNN_ACT_SELU: return kSeluScale * (x > 0.0f ? x : kSeluAlpha * expm1f(x));
    case TFGNN_ACT_GELU: {
      // tf2_gnn/utils/activation.py:7-14 (tanh approximation)
      const float c = 0.7978845608028654f;  // sqrt(2/pi)
      float cdf = 0.5f * (1.0f + tanhf(c * (x + 0.044715f * x * x * x)));
      return x * cdf;
    }
    case TFGNN_ACT_SIGMOID: return 1.0f / (1.0f + expf(-x));
    default: return x;
  }
}

// act'(x) from the OUTPUT y = act(x), for every activation but gelu
__device__ __forceinline__ float act_grad_from_output(float y, int act) {
  switch (act) {
    case TFGNN_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case TFGNN_ACT_TANH: return 1.f - y * y;
    case TFGNN_ACT_LEAKY_RELU: return y > 0.f ? 1.f : kLeakyReluAlpha;
    case TFGNN_ACT_ELU: return y > 0.f ? 1.f : y + 1.f;                               // d/dx (e^x - 1) = y + 1
    case TFGNN_ACT_SELU: return y > 0.f ? kSeluScale : y + kSeluScale * kSeluAlpha;   // scale*alpha*e^x = y + scale*alpha
    case TFGNN_ACT_SIGMOID: return y * (1.f - y);
    default: return 1.f;
  }
}
// gelu (tanh approximation) is not invertible from its output: its derivative comes from the PRE-activation x
__device__ __forceinline__ float gelu_grad_from_input(float x) {
  const float c = 0.7978845608028654f;
  const float t = tanhf(c * (x + 0.044715f * x * x * x));
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * c * (1.0f + 3.0f * 0.044715f * x * x);
}

template <int ACT>
__device__ __forceinline__ float apply_act_t(float x) {
  return apply_act(x, ACT);
}

// Activation of N register values with the switch hoisted OUT of the element loop: only the selected
// case's (short) loop is ever fetched.  Inlining apply_act() per element put every libdevice expansion
// (tanhf, expm1f, ...) N times into the epilogue: ~80 KB of straight-line SASS that thrashed the
// instruction cache (measured: ~30 us per 128x128 output tile in the tensor-core GEMM epilogue).  The transcendental
// cases therefore go through ONE out-of-line copy - which takes and returns VALUES: an out-of-line function
// over `float*` (round 1) made the caller's array addressable, so every epilogue kept its chunk in LOCAL
// memory (STL/LDL around each chunk, also on the relu path; 17-20 us per 128x256 tile in the fused kernel).
static __device__ __noinline__ float4 apply_act_slow4(float4 x, int act) {
  return make_float4(apply_act(x.x, act), apply_act(x.y, act), apply_act(x.z, act), apply_act(x.w, act));
}
static __device__ __noinline__ float apply_act_slow1(float x, int act) { return apply_act(x, act); }
template <int N>
__device__ __forceinline__ void apply_act_vec(float (&v)[N], int act) {
  if (act == TFGNN_ACT_NONE) return;
  if (act == TFGNN_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = fmaxf(v[j], 0.0f);
  } else if (act == TFGNN_ACT_LEAKY_RELU) {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = v[j] > 0.0f ? v[j] : kLeakyReluAlpha * v[j];
  } else if constexpr (N % 4 == 0) {
#pragma unroll
    for (int j = 0; j < N; j += 4) {
      const float4 r = apply_act_slow4(make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]), act);
      v[j] = r.x; v[j + 1] = r.y; v[j + 2] = r.z; v[j + 3] = r.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = apply_act_slow1(v[j], act);
  }
}

__device__ __forceinline__ float4 ldg_f4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

struct PtrTable {
  const void* p[TFGNN_MAX_EDGE_TYPES];
};
struct CountTable {
  long long n[TFGNN_MAX_EDGE_TYPES];
};

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// Blocks of 256 threads for a grid-stride loop over n items: at most 32 per SM of the H100's 132.
inline int grid_for(long long n) {
  const int g = ceil_div(n, 256);
  return g < 1 ? 1 : (g > 132 * 32 ? 132 * 32 : g);
}

}  // namespace tfgnn

// The opaque batch (see include/tfgnn_b200.h).  Keyed CSR: segment s = l*V + v holds the
// sources of all type-l edges into v, so c[l,v] = row_ptr[s+1]-row_ptr[s].
struct tfgnn_batch {
  long long V = 0;        // number of TARGET nodes owned by this batch (= rows of every layer output)
  long long V_src = 0;    // number of rows of the source node table (== V unless target-range sharded)
  long long tgt_off = 0;  // global id of local target 0 (target-range sharding, SURVEY.md §8e)
  // TFGNN_PREPARE_TRANSPOSE_OWNED: segments are (type, global source) over V = V_src nodes, values are local target ids of
  // the owned range [own_begin, own_begin + own_count)
  bool owned_transpose = false;
  long long own_begin = 0, own_count = 0;
  int L = 0;
  long long M_in = 0;     // edges handed in
  int device = 0;
  int32_t* row_ptr = nullptr;     // [L*V+1]
  int32_t* src_sorted = nullptr;  // [M_in] (first row_ptr[L*V] entries valid)
  int32_t* invalid_count = nullptr;
  // caller-owned adjacency (kept for the TFGNN_PATH_ATOMIC evidence path only)
  const int32_t* adj[TFGNN_MAX_EDGE_TYPES] = {};
  long long E[TFGNN_MAX_EDGE_TYPES] = {};
  // the stream the batch was last used on: allocations / frees of its buffers are ordered on it.  A batch may move
  // between streams from one call to the next (batch_enter orders the new stream after the old one), but it must
  // not be used from two streams or two host threads at the same time.
  cudaStream_t cur_stream = nullptr;
  bool used = false;
  // tfgnn_b200_rgcn_fwd_allgather: peer copies of the output table the fused kernel's epilogue also stores to (set for the
  // duration of that call only)
  float* peer_out[TFGNN_MAX_PEERS] = {};
  int n_peer_out = 0;
  float* mc_out = nullptr;   // multicast mapping of all replicas (one multimem.st reaches every GPU)
  // tfgnn_b200_rgcn_ln_fwd: LayerNormalization parameters for the fused epilogue (set for the duration of that call only)
  const float* ln_gamma = nullptr;
  const float* ln_beta = nullptr;
  float ln_eps = 0.f;
  cudaEvent_t ev_switch = nullptr;
  // internal fork/join streams of the gather || node-GEMM pipeline (created lazily)
  static constexpr int kPipeBufs = 3;
  bool pipe_ready = false;
  cudaStream_t pipe_gather = nullptr, pipe_gemm = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join_g = nullptr, ev_join_m = nullptr;
  cudaEvent_t ev_g[kPipeBufs] = {}, ev_m[kPipeBufs] = {};
};

namespace tfgnn {
// Every entry point that takes a batch calls this first: binds the batch to `st` for this call.
int batch_enter(tfgnn_batch* b, cudaStream_t st);
// Stream-ordered device memory from the library's PRIVATE cudaMemPool (release threshold = keep everything:
// after the first batches no call on the per-batch path reaches cudaMalloc / cudaFree or synchronises).
int pool_alloc(void** p, size_t bytes, cudaStream_t st);
void pool_free(void* p, cudaStream_t st);

// A buffer from the library pool, freed (stream-ordered, after the work queued so far) when it goes out of scope.  Every
// temporary of a layer call is one, owned by the narrowest scope that covers its uses: a nested call cannot free or
// regrow a buffer its caller still holds.  Move-only: it owns its pointer.
struct PoolBuffer {
  cudaStream_t st;
  void* p = nullptr;
  explicit PoolBuffer(cudaStream_t s) : st(s) {}
  PoolBuffer(PoolBuffer&& o) noexcept : st(o.st), p(o.p) { o.p = nullptr; }
  PoolBuffer(const PoolBuffer&) = delete;
  PoolBuffer& operator=(const PoolBuffer&) = delete;
  ~PoolBuffer() { pool_free(p, st); }
  int alloc(size_t bytes) { return pool_alloc(&p, bytes, st); }
  float* f() const { return (float*)p; }
};
}  // namespace tfgnn
