// One optimizer step over all variables of a model (graph_task_model.py:224-324): Keras SGD / RMSprop / Adam
// (optimizer_v2, epsilon 1e-7, beta_1 0.9, beta_2 0.999) after clip-by-value, clip-by-norm or clip-by-global-norm.
//
// Every tensor is cut into chunks of kOptChunk elements and the chunks of all tensors are numbered in tensor order; CTA b
// updates chunk b.  The per-tensor table (pointers, size, first chunk) goes to the device through the call's pool buffer, so
// one launch updates every tensor whatever their number.  Norm clipping runs one reduction launch first: CTA b writes the
// sum of squares of chunk b (fixed tree order).  Each update CTA then combines the partials it needs (its tensor's chunks in
// chunk order; for the global norm every tensor's sum, in tensor order) into the clip scale on the device: no host round
// trip, and the same gradients give the same bits on every call and on every rank that holds them.
#include <math.h>

#include <vector>

#include "layers.cuh"

namespace tfgnn {

constexpr int kOptThreads = 256;
constexpr int kOptChunk = 4096;   // elements per CTA (a constant: the norms must not depend on the grid)
constexpr float kAdamBeta1 = 0.9f, kAdamBeta2 = 0.999f;   // Keras defaults, float32 tensors in TF's training ops

struct OptTensor {
  float* w;
  const float* g;
  float* a;
  float* b;
  long long n;
  long long chunk0;   // first chunk of this tensor; the table holds one more entry whose chunk0 is the total
};

struct OptArgs {
  int kind, clip_mode, n;
  float lr, momentum, rho, alpha, c;
};

__device__ __forceinline__ int tensor_of_chunk(const OptTensor* __restrict__ tab, int n, long long chunk) {
  int lo = 0, hi = n - 1;   // last tensor with chunk0 <= chunk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ float cta_sum_f(float v) {
  __shared__ float s[kOptThreads];
  __syncthreads();   // the buffer may still be read from a previous call
  s[threadIdx.x] = v;
  __syncthreads();
  for (int k = kOptThreads / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) s[threadIdx.x] += s[threadIdx.x + k];
    __syncthreads();
  }
  return s[0];
}

// sum of squares of one chunk -> partial[chunk]
__global__ void __launch_bounds__(kOptThreads)
opt_sumsq_kernel(const OptTensor* __restrict__ tab, int n, float* __restrict__ partial) {
  const long long chunk = blockIdx.x;
  const OptTensor t = tab[tensor_of_chunk(tab, n, chunk)];
  const long long beg = (chunk - t.chunk0) * kOptChunk;
  const long long end = beg + kOptChunk < t.n ? beg + kOptChunk : t.n;
  float s = 0.f;
  for (long long i = beg + threadIdx.x; i < end; i += kOptThreads) {
    const float g = __ldg(t.g + i);
    s += g * g;
  }
  s = cta_sum_f(s);
  if (threadIdx.x == 0) partial[chunk] = s;
}

// sum of the partials [c0, c1) in a fixed order (thread j: c0 + j, c0 + j + kOptThreads, ...; then the tree)
__device__ __forceinline__ float sum_partials(const float* __restrict__ partial, long long c0, long long c1) {
  float s = 0.f;
  for (long long c = c0 + threadIdx.x; c < c1; c += kOptThreads) s += partial[c];
  return cta_sum_f(s);
}

__global__ void __launch_bounds__(kOptThreads)
opt_update_kernel(const OptTensor* __restrict__ tab, OptArgs a, const float* __restrict__ partial) {
  const long long chunk = blockIdx.x;
  const int ti = tensor_of_chunk(tab, a.n, chunk);
  const OptTensor t = tab[ti];
  float scale = 1.f;
  if (a.clip_mode == TFGNN_CLIP_NORM) {
    // tf.clip_by_norm: g * c / max(||g||, c)
    const float norm = sqrtf(sum_partials(partial, t.chunk0, tab[ti + 1].chunk0));
    scale = fmaxf(norm, a.c);
  } else if (a.clip_mode == TFGNN_CLIP_GLOBAL_NORM) {
    // tf.clip_by_global_norm: per-tensor sums of squares, added in tensor order; c * min(1 / gn, 1 / c), NaN if gn is not
    // finite
    float total = 0.f;
    for (int j = 0; j < a.n; ++j) total += sum_partials(partial, tab[j].chunk0, tab[j + 1].chunk0);
    const float gn = sqrtf(total);
    scale = a.c * fminf(1.f / gn, 1.f / a.c) + (gn - gn);
  }
  const long long beg = (chunk - t.chunk0) * kOptChunk;
  const long long end = beg + kOptChunk < t.n ? beg + kOptChunk : t.n;
  for (long long i = beg + threadIdx.x; i < end; i += kOptThreads) {
    float g = __ldg(t.g + i);
    if (a.clip_mode == TFGNN_CLIP_VALUE) g = fminf(fmaxf(g, -a.c), a.c);
    else if (a.clip_mode == TFGNN_CLIP_NORM) g = g * a.c / scale;
    else if (a.clip_mode == TFGNN_CLIP_GLOBAL_NORM) g = g * scale;
    float w = t.w[i];
    if (a.kind == TFGNN_OPT_SGD) {
      if (t.a) {                                       // ResourceApplyKerasMomentum
        const float acc = t.a[i] * a.momentum - a.lr * g;
        t.a[i] = acc;
        w += acc;
      } else {                                         // ResourceApplyGradientDescent
        w -= a.lr * g;
      }
    } else if (a.kind == TFGNN_OPT_RMSPROP) {
      float ms = t.a[i];
      ms += (g * g - ms) * (1.f - a.rho);
      t.a[i] = ms;
      if (t.b) {                                       // ResourceApplyRMSProp
        const float mom = a.momentum * t.b[i] + a.lr * g / sqrtf(ms + kSmallNumber);
        t.b[i] = mom;
        w -= mom;
      } else {
        w -= a.lr * g / (sqrtf(ms) + kSmallNumber);
      }
    } else {                                           // ResourceApplyAdam
      float m = t.a[i], v = t.b[i];
      m += (g - m) * (1.f - kAdamBeta1);
      v += (g * g - v) * (1.f - kAdamBeta2);
      t.a[i] = m;
      t.b[i] = v;
      w -= a.alpha * m / (sqrtf(v) + kSmallNumber);
    }
    t.w[i] = w;
  }
}

}  // namespace tfgnn

using namespace tfgnn;

extern "C" int tfgnn_b200_optimizer_step(int32_t kind, int32_t num_tensors, float* const* params, const float* const* grads,
                                         float* const* slot_a, float* const* slot_b, const int64_t* sizes, float lr,
                                         float momentum, float rho, int64_t step, int32_t clip_mode, float clip,
                                         void* stream) {
  TFGNN_REQUIRE(kind == TFGNN_OPT_SGD || kind == TFGNN_OPT_RMSPROP || kind == TFGNN_OPT_ADAM,
                "tfgnn_b200_optimizer_step: unknown optimizer kind");
  TFGNN_REQUIRE(clip_mode >= TFGNN_CLIP_NONE && clip_mode <= TFGNN_CLIP_GLOBAL_NORM,
                "tfgnn_b200_optimizer_step: unknown clip mode");
  TFGNN_REQUIRE(num_tensors >= 0 && step >= 0, "tfgnn_b200_optimizer_step: negative num_tensors or step");
  if (num_tensors == 0) return 0;
  TFGNN_REQUIRE(params && grads && sizes, "tfgnn_b200_optimizer_step: NULL params, grads or sizes");
  // slots: SGD a = momentum accumulator (momentum > 0); RMSprop a = mean square, b = momentum (momentum > 0); Adam a = m, b = v
  const bool need_a = kind != TFGNN_OPT_SGD || momentum > 0.f;
  const bool need_b = kind == TFGNN_OPT_ADAM || (kind == TFGNN_OPT_RMSPROP && momentum > 0.f);
  TFGNN_REQUIRE((!need_a || slot_a) && (!need_b || slot_b), "tfgnn_b200_optimizer_step: NULL slot table");
  std::vector<OptTensor> tab((size_t)num_tensors + 1);
  long long chunks = 0;
  for (int i = 0; i < num_tensors; ++i) {
    TFGNN_REQUIRE(sizes[i] >= 0, "tfgnn_b200_optimizer_step: negative tensor size");
    OptTensor& t = tab[i];
    t.n = sizes[i];
    t.chunk0 = chunks;
    t.w = params[i];
    t.g = grads[i];
    t.a = need_a ? slot_a[i] : nullptr;
    t.b = need_b ? slot_b[i] : nullptr;
    TFGNN_REQUIRE(t.n == 0 || (t.w && t.g && (!need_a || t.a) && (!need_b || t.b)),
                  "tfgnn_b200_optimizer_step: NULL parameter, gradient or slot pointer");
    chunks += (t.n + kOptChunk - 1) / kOptChunk;
  }
  tab[num_tensors] = OptTensor{nullptr, nullptr, nullptr, nullptr, 0, chunks};
  TFGNN_REQUIRE(chunks < (1ll << 31), "tfgnn_b200_optimizer_step: too many elements");
  if (chunks == 0) return 0;
  OptArgs a;
  a.kind = kind;
  a.clip_mode = clip_mode;
  a.n = num_tensors;
  a.lr = lr;
  a.momentum = momentum;
  a.rho = rho;
  a.c = clip;
  // Adam: alpha = lr sqrt(1 - beta_2^t) / (1 - beta_1^t), t = step + 1 (Keras' iterations + 1), on the float32 betas the
  // update uses
  const double t = (double)step + 1.0;
  a.alpha = (float)((double)lr * sqrt(1.0 - pow((double)kAdamBeta2, t)) / (1.0 - pow((double)kAdamBeta1, t)));
  cudaStream_t st = (cudaStream_t)stream;
  PoolBuffer dtab{st}, partial{st};
  int rc = dtab.alloc(tab.size() * sizeof(OptTensor));
  if (rc) return rc;
  TFGNN_CUDA(cudaMemcpyAsync(dtab.p, tab.data(), tab.size() * sizeof(OptTensor), cudaMemcpyHostToDevice, st));
  const OptTensor* d_tab = (const OptTensor*)dtab.p;
  if (clip_mode == TFGNN_CLIP_NORM || clip_mode == TFGNN_CLIP_GLOBAL_NORM) {
    rc = partial.alloc((size_t)chunks * sizeof(float));
    if (rc) return rc;
    opt_sumsq_kernel<<<(unsigned)chunks, kOptThreads, 0, st>>>(d_tab, num_tensors, partial.f());
    TFGNN_LAUNCH_CHECK();
  }
  opt_update_kernel<<<(unsigned)chunks, kOptThreads, 0, st>>>(d_tab, a, partial.f());
  TFGNN_LAUNCH_CHECK();
  return 0;
}
