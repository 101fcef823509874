// Shared helpers for the rave_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/rave_b200.h"

namespace rave {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);

#define RAVE_CHECK_ARG(cond, ...)                \
  do {                                           \
    if (!(cond)) {                               \
      rave::set_error(__VA_ARGS__);              \
      return 1;                                  \
    }                                            \
  } while (0)

#define RAVE_CHECK_LAUNCH(name)                                              \
  do {                                                                       \
    cudaError_t e__ = cudaGetLastError();                                    \
    if (e__ != cudaSuccess) {                                                \
      rave::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return 2;                                                              \
    }                                                                        \
    rave::count_launch();                                                    \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Deterministic cross-block sums: out[g * n + i] += sum of the partials i of the blocks of group g, added in block order.
// A group is the set of blocks sharing one index along grid dimension `gdim` (0 = x, 1 = y; -1: one group, the whole
// grid).  Float atomics would add the partials in arrival order, which changes the last bits from run to run -- and a
// training run amplifies such differences step after step.  Each launch gets its own stream-ordered scratch (partials +
// arrival counter, graph-capturable); every block stores its n partials, the last block to arrive adds them up.
struct BlockSum {
  float *part;        // [blocks][n]
  unsigned *ticket;
  int n, gdim;
  int limit;          // outputs beyond out[limit - 1] are dropped (last group of a partial channel tile)
};
inline int block_sum_begin(BlockSum *s, long blocks, int n, cudaStream_t stream, int gdim = -1) {
  void *p = nullptr;
  if (cudaMallocAsync(&p, 16 + (size_t)blocks * n * sizeof(float), stream) != cudaSuccess) {
    set_error("block_sum: cudaMallocAsync of %ld x %d partials failed", blocks, n);
    return 2;
  }
  cudaMemsetAsync(p, 0, 16, stream);
  s->ticket = reinterpret_cast<unsigned *>(p);
  s->part = reinterpret_cast<float *>(reinterpret_cast<char *>(p) + 16);
  s->n = n;
  s->gdim = gdim;
  s->limit = 0x7fffffff;
  return 0;
}
inline void block_sum_end(const BlockSum &s, cudaStream_t stream) { cudaFreeAsync(s.ticket, stream); }

__device__ __forceinline__ unsigned block_linear_id() {
  return blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
}
// partial i of this block (one thread per i)
__device__ __forceinline__ void block_sum_put(const BlockSum &s, int i, float v) {
  s.part[(size_t)block_linear_id() * s.n + i] = v;
}
// called by every thread of every block after its block_sum_put calls; true (in all threads of the block) in the last
// block, whose out[] writes are then complete and visible to the whole block
__device__ __forceinline__ bool block_sum_finish(const BlockSum &s, float *out) {
  __shared__ unsigned is_last;
  __threadfence();
  __syncthreads();
  const unsigned gx = gridDim.x, gy = gridDim.y, nb = gx * gy * gridDim.z;
  if (threadIdx.x == 0) is_last = atomicAdd(s.ticket, 1u) == nb - 1 ? 1u : 0u;
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  const unsigned groups = s.gdim == 0 ? gx : s.gdim == 1 ? gy : 1u, per = nb / groups;
  const unsigned total = min(groups * (unsigned)s.n, (unsigned)s.limit);
  for (unsigned o = threadIdx.x; o < total; o += blockDim.x) {
    const unsigned g = o / s.n, i = o % s.n;
    float t = 0.f;
    for (unsigned j = 0; j < per; ++j) {
      const unsigned b = s.gdim == 0 ? g + gx * j : s.gdim == 1 ? (j % gx) + gx * (g + gy * (j / gx)) : j;
      t += __ldcg(s.part + (size_t)b * s.n + i);
    }
    out[o] += t;
  }
  __syncthreads();
  return true;
}

// VariationalEncoder.reparametrize's sample minus the latent mean: eps (softplus(scale) + 1e-4) + mean - latent_mean,
// torch's softplus (threshold 20), every step rounded on its own (no FMA contraction).  Shared by the prior's latent
// classes and the exported model's latent projection, so both see the same bits.
__device__ __forceinline__ float centred_sample(float mean, float scale, float eps, float latent_mean) {
  const float sd = __fadd_rn(scale > 20.f ? scale : log1pf(expf(scale)), 1e-4f);
  return __fsub_rn(__fadd_rn(__fmul_rn(eps, sd), mean), latent_mean);
}

// activation(dim) of rave/blocks.py: LeakyReLU(slope) / Snake(alpha)
__device__ __forceinline__ float act_apply(float x, int act, float slope, float alpha) {
  if (act == RAVE_ACT_LEAKY) return x > 0.f ? x : x * slope;
  if (act == RAVE_ACT_SNAKE) {
    float s = sinf(alpha * x);
    return x + s * s / (alpha + 1e-9f);
  }
  return x;
}
__device__ __forceinline__ float act_grad(float x, int act, float slope, float alpha) {
  if (act == RAVE_ACT_LEAKY) return x > 0.f ? 1.f : slope;
  if (act == RAVE_ACT_SNAKE) {
    // d/dx [x + sin^2(a x)/(a+eps)] = 1 + a sin(2 a x)/(a+eps)
    return 1.f + alpha * sinf(2.f * alpha * x) / (alpha + 1e-9f);
  }
  return 1.f;
}

}  // namespace rave
