// Exponential moving average of a model's parameters (the reference's EMA callback, scripts/train.py:81-119) as one
// multi-tensor launch, and the in-place exchange of parameters and averages (its swap_weights).
//
// The tensors are described by a device table built once by the caller (the addresses are stable):
//   table = [ p[T] | ema[T] | numel[T] | chunk0[T + 1] ]   (int64; p and ema are float32 pointers)
// Tensor t owns chunks [chunk0[t], chunk0[t + 1]) of kEmaChunk elements; a CTA walks the chunks grid-stride and finds
// each chunk's tensor by binary search in chunk0.  Within a chunk the threads use float4 accesses when p and ema have
// the same 16-byte misalignment (scalar head, vector body, scalar tail), scalar accesses otherwise.  Every element is
// read and written by one thread, with no reduction: the output does not depend on the schedule.
//
// Arithmetic contract: ema = rn(rn(ema * f) + rn(p * g)), f = float32(factor), g = float32(1 - factor) with 1 - factor
// in double on the host -- what torch computes for `w * factor + p * (1 - factor)` on float32 tensors.  Spelled with
// __fmul_rn / __fadd_rn so that nvcc cannot contract it into an FMA.
//
// state = [ initialised[T] | ticket ] (int32).  While initialised[t] is 0 the update copies p into ema instead of
// averaging (the reference's first call, which clones).  The flags are read by every CTA and set only by the last CTA
// to finish (a completion ticket), so no CTA of the same launch can see a flag change: the decision lives on the
// device and a CUDA graph can capture it.
#include "common.cuh"

namespace rave {

constexpr int kEmaThreads = 256;
constexpr int kEmaVec = 4;                                   // float4
constexpr int kEmaPer = 4;                                   // float4 per thread per chunk
constexpr long long kEmaChunk = (long long)kEmaThreads * kEmaVec * kEmaPer;

struct EmaTable {
  float *const *p;
  float *const *ema;
  const long long *numel;
  const long long *chunk0;
  int T;
};

__device__ __forceinline__ EmaTable ema_table(const long long *table, int T) {
  EmaTable tb;
  tb.p = reinterpret_cast<float *const *>(table);
  tb.ema = reinterpret_cast<float *const *>(table + T);
  tb.numel = table + 2 * T;
  tb.chunk0 = table + 3 * T;
  tb.T = T;
  return tb;
}

// the tensor owning chunk c: the last t with chunk0[t] <= c
__device__ __forceinline__ int ema_tensor_of(const EmaTable &tb, long long c) {
  int lo = 0, hi = tb.T - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tb.chunk0[mid] <= c) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct EmaUpdateOp {
  float f, g;
  int init;
  __device__ __forceinline__ void operator()(float &p, float &e) const {
    e = init ? __fadd_rn(__fmul_rn(e, f), __fmul_rn(p, g)) : p;
  }
};
struct EmaSwapOp {
  __device__ __forceinline__ void operator()(float &p, float &e) const {
    const float t = p;
    p = e;
    e = t;
  }
};

// apply op to elements [0, n) of (p, e); writes p only when WriteP
template <bool WriteP, class Op>
__device__ __forceinline__ void ema_chunk(float *p, float *e, int n, const Op &op) {
  const unsigned mp = (unsigned)(reinterpret_cast<uintptr_t>(p) & 15u);
  const unsigned me = (unsigned)(reinterpret_cast<uintptr_t>(e) & 15u);
  int head = n, body = 0;
  if (mp == me) {
    head = min(n, (int)(((16u - mp) & 15u) >> 2));
    body = (n - head) / kEmaVec;
  }
  for (int i = threadIdx.x; i < head; i += kEmaThreads) {
    float a = p[i], b = e[i];
    op(a, b);
    if (WriteP) p[i] = a;
    e[i] = b;
  }
  float4 *p4 = reinterpret_cast<float4 *>(p + head);
  float4 *e4 = reinterpret_cast<float4 *>(e + head);
  float4 a[kEmaPer], b[kEmaPer];
#pragma unroll
  for (int k = 0; k < kEmaPer; ++k) {
    const int i = threadIdx.x + k * kEmaThreads;
    if (i < body) {
      a[k] = p4[i];
      b[k] = e4[i];
    }
  }
#pragma unroll
  for (int k = 0; k < kEmaPer; ++k) {
    const int i = threadIdx.x + k * kEmaThreads;
    if (i < body) {
      op(a[k].x, b[k].x);
      op(a[k].y, b[k].y);
      op(a[k].z, b[k].z);
      op(a[k].w, b[k].w);
      if (WriteP) p4[i] = a[k];
      e4[i] = b[k];
    }
  }
  for (int i = head + body * kEmaVec + threadIdx.x; i < n; i += kEmaThreads) {
    float x = p[i], y = e[i];
    op(x, y);
    if (WriteP) p[i] = x;
    e[i] = y;
  }
}

__global__ void __launch_bounds__(kEmaThreads) ema_update_kernel(const long long *table, int T, long long n_chunks,
                                                                 int *state, float f, float g) {
  const EmaTable tb = ema_table(table, T);
  for (long long c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = ema_tensor_of(tb, c);
    const long long s = (c - tb.chunk0[t]) * kEmaChunk;
    const int n = (int)min(kEmaChunk, tb.numel[t] - s);
    ema_chunk<false>(tb.p[t] + s, tb.ema[t] + s, n, EmaUpdateOp{f, g, state[t]});
  }
  // completion ticket: the last CTA sets every flag, after every CTA has read the flags it needed
  __shared__ unsigned last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(reinterpret_cast<unsigned *>(state + T), 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  for (int t = threadIdx.x; t < T; t += kEmaThreads) state[t] = 1;
  if (threadIdx.x == 0) state[T] = 0;
}

__global__ void __launch_bounds__(kEmaThreads) ema_swap_kernel(const long long *table, int T, long long n_chunks) {
  const EmaTable tb = ema_table(table, T);
  for (long long c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = ema_tensor_of(tb, c);
    const long long s = (c - tb.chunk0[t]) * kEmaChunk;
    const int n = (int)min(kEmaChunk, tb.numel[t] - s);
    ema_chunk<true>(tb.p[t] + s, tb.ema[t] + s, n, EmaSwapOp{});
  }
}

static int ema_grid(long long n_chunks) {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return (int)min(n_chunks, (long long)sms * 8);
}

}  // namespace rave

extern "C" long long rave_ema_chunk_elems(void) { return rave::kEmaChunk; }

extern "C" int rave_ema_update(const long long *table, int n_tensors, long long n_chunks, int *state, float factor,
                               float one_minus_factor, void *stream) {
  RAVE_CHECK_ARG(table && state && n_tensors > 0 && n_chunks > 0, "rave_ema_update: bad table (T=%d, chunks=%lld)",
                 n_tensors, n_chunks);
  rave::ema_update_kernel<<<rave::ema_grid(n_chunks), rave::kEmaThreads, 0, (cudaStream_t)stream>>>(
      table, n_tensors, n_chunks, state, factor, one_minus_factor);
  RAVE_CHECK_LAUNCH("rave_ema_update");
  return 0;
}

extern "C" int rave_ema_swap(const long long *table, int n_tensors, long long n_chunks, void *stream) {
  RAVE_CHECK_ARG(table && n_tensors > 0 && n_chunks > 0, "rave_ema_swap: bad table (T=%d, chunks=%lld)",
                 n_tensors, n_chunks);
  rave::ema_swap_kernel<<<rave::ema_grid(n_chunks), rave::kEmaThreads, 0, (cudaStream_t)stream>>>(table, n_tensors,
                                                                                                 n_chunks);
  RAVE_CHECK_LAUNCH("rave_ema_swap");
  return 0;
}
