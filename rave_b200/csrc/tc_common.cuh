// Raw PTX wrappers for the Hopper (sm_90a) tensor-core path: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence /
// commit / wait, shared-memory matrix descriptors) and the shared-memory accumulator hand-over between the MMA
// warpgroup and the epilogue warps.  Bit layouts follow the PTX ISA "Matrix Descriptor Format" of wgmma (the fields
// CUTLASS' cute::GMMA::GmmaDescriptor exposes).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <utility>

#include "common.cuh"
#include "wgmma_sm90.cuh"

namespace rave {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a mis-programmed pipeline traps (the launch fails with an error) instead of hanging the GPU.  No
// printf by default: a function call anywhere in a kernel makes ptxas serialise every wgmma of it (warning C7510: a wait
// for completion after each m64nNk16), which costs the tensor pipe most of its overlap.  Building with
// -DRAVE_MBAR_DEBUG prints the block and thread of a timed-out wait before the trap (slow kernels, diagnosis only).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > 20000000u) {
#ifdef RAVE_MBAR_DEBUG
      printf("rave_b200: mbarrier wait timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x);
#endif
      __trap();
    }
  }
}

// 32-byte row segments (32-byte aligned) as two 128-bit accesses
__device__ __forceinline__ void ldg256(const void *p, uint32_t *r) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "l"(p));
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
               : "l"(reinterpret_cast<const uint8_t *>(p) + 16));
}
__device__ __forceinline__ void stg256(void *p, const uint32_t *r) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(reinterpret_cast<uint8_t *>(p) + 16), "r"(r[4]), "r"(r[5]),
               "r"(r[6]), "r"(r[7])
               : "memory");
}

// One lane of a fully converged warp.  The producer loops run WARP-UNIFORM (all 32 lanes execute the loop, only the
// TMA instructions are predicated on the elected lane): stage indices, shared-memory addresses and coordinates then
// live in uniform registers instead of being broadcast from one lane per instruction.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *smem, const CUtensorMap *m, uint64_t *bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void *smem, const CUtensorMap *m, uint64_t *bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// 3-D tiled loads / stores of epilogue operand chunks (channel, row, batch): CTA-local barrier, bulk-group stores
__device__ __forceinline__ void tma_load_3d(void *smem, const CUtensorMap *m, uint64_t *bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap *m, const void *smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(m),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *m, const void *smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {      // at most N bulk groups still READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void sts128(void *p, const uint32_t *r) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(smem_u32(p)), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// ------------------------------------------------------------------ wgmma (sm_90a)
// One warpgroup (4 warps, 128 threads) issues every MMA of a 128-row tile as two m64 halves and holds the fp32
// accumulators in registers: d[h][N/2] for rows 64 h .. 64 h + 63.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Register rebalancing between warpgroups (every thread of the warpgroup executes it): a producer warpgroup gives
// registers back so that the MMA warpgroups of the same CTA can grow past the launch-time share.  N is a multiple of 8.
template <int N>
__device__ __forceinline__ void warpgroup_reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void warpgroup_reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float *d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Accumulator hand-over.  The warps of an epilogue own one ROW of a 128-row tile each (thread = row quad * 32 + lane)
// and read consecutive columns; wgmma leaves row pieces spread over the lanes of its warpgroup.  The MMA warpgroup
// therefore stores a finished tile to a shared-memory buffer [128][ld] fp32 (ld = 4 mod 32 words: the 8 lanes of a
// 16-byte-load phase hit disjoint banks) and the epilogue reads it back with acc_ld.  An accumulator address is
// (row << 16) | column, relative to the buffer set by acc_bind.
static __shared__ uint32_t s_acc_addr, s_acc_ld;
__host__ __device__ constexpr int acc_pitch(int cols) { return (cols + 31) / 32 * 32 + 4; }
__device__ __forceinline__ void acc_bind(const void *buf, int ld) {    // one thread, before the block-wide barrier
  s_acc_addr = smem_u32(buf);
  s_acc_ld = (uint32_t)ld;
}
// store the warpgroup's accumulators of a 128 x N tile (wgmma fragment: d[4j + {0,1}] at row 16 warp + lane / 4,
// columns 8 j + 2 (lane % 4) + {0,1}; d[4j + {2,3}] eight rows further down) at column `col0` and row `row0` of the
// buffer (row0 = 128: the second of two accumulator buffers bound back to back)
template <int N>
__device__ __forceinline__ void acc_store(const float (*d)[N / 2], int wg_thread, int col0 = 0, int row0 = 0) {
  const int w = wg_thread >> 5, l = wg_thread & 31;
  const uint32_t ld = s_acc_ld;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t r0 = (uint32_t)(row0 + 64 * h + 16 * w + (l >> 2));
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const uint32_t c = (uint32_t)(col0 + 8 * j + 2 * (l & 3));
      const uint32_t a0 = s_acc_addr + (r0 * ld + c) * 4u, a1 = a0 + 8u * ld * 4u;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0), "f"(d[h][4 * j]), "f"(d[h][4 * j + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a1), "f"(d[h][4 * j + 2]), "f"(d[h][4 * j + 3]) : "memory");
    }
  }
}
// NC consecutive fp32 accumulators of row (taddr >> 16) + lane, from column taddr & 0xFFFF
template <int NC>
__device__ __forceinline__ void acc_ld(uint32_t taddr, float *v) {
  const uint32_t row = (taddr >> 16) + (threadIdx.x & 31), col = taddr & 0xFFFFu;
  const uint32_t a = s_acc_addr + (row * s_acc_ld + col) * 4u;
#pragma unroll
  for (int i = 0; i < NC / 4; ++i)
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v[4 * i]), "=f"(v[4 * i + 1]), "=f"(v[4 * i + 2]), "=f"(v[4 * i + 3])
                 : "r"(a + 16u * i)
                 : "memory");
}

// Stores the warpgroup's 128 x BLOCK_N accumulator tile (wgmma fragment layout, see acc_store) into dst rows m0 ..
// (row pitch Cn, columns from n0), clipped to Cm x Cn.  Cn is a multiple of 8, so a fragment pair is valid as a whole.
template <int BLOCK_N>
__device__ __forceinline__ void store_wgrad_tile(const float (*d)[BLOCK_N / 2], float *dst, int m0, int n0, int Cm,
                                                 int Cn) {
  const int w = (threadIdx.x & 127) >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int m = m0 + 64 * h + 16 * w + (l >> 2) + 8 * r;
      if (m >= Cm) continue;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (l & 3);
        if (n < Cn)
          *reinterpret_cast<float2 *>(dst + (size_t)m * Cn + n) = make_float2(d[h][4 * j + 2 * r], d[h][4 * j + 2 * r + 1]);
      }
    }
  }
}

// Bias gradient of the weight-gradient kernels: the column-sum CTAs of every split-K slice write their partial sums to
// part[split][m] (no atomics: the slices would add in arrival order), this kernel adds them up in slice order.
template <int UNUSED = 0>
__global__ void __launch_bounds__(256) dbias_sum_kernel(const float *__restrict__ part, float *__restrict__ dbias,
                                                        int splits, int pitch, int Cm) {
  const int m = blockIdx.x * 256 + threadIdx.x;
  if (m >= Cm) return;
  float t = 0.f;
  for (int s = 0; s < splits; ++s) t += part[(size_t)s * pitch + m];
  dbias[m] += t;
}

// ------------------------------------------------------------------ programmatic dependent launch
// Every tensor-core kernel finishes its prologue (barrier init, tensor-map prefetch) and then WAITS for the
// grids it depends on (griddepcontrol.wait: full completion + memory flush of the previous kernels in the stream); it
// also lets its own dependents start early (launch_dependents).  Launched with the programmatic-stream-serialization
// attribute (launch_pdl), the next kernel's CTAs take SMs as soon as this one's CTAs leave them, so its launch latency
// and prologue overlap this kernel's tail -- a chain of ~50 short kernels (the encoder / generator forward) otherwise
// pays ~3-4 us of ramp per launch.  Nothing before the wait touches global memory another kernel writes.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args &&...args) {
#ifndef __CUDA_ARCH__
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
#else
  return cudaSuccess;
#endif
}

// Grid of a persistent kernel: one CTA per SM, fewer when there are fewer tiles.
static inline int persistent_grid(int tiles) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return tiles < sms ? tiles : sms;
}

// launch_pdl of Kernel with `smem` bytes of dynamic shared memory (the opt-in is raised once per new maximum of the
// instance); 0 = launched, 2 = CUDA error (message under `name`).
template <auto Kernel, typename... Args>
static int launch_tc(const char *name, int grid, int threads, int smem, cudaStream_t stream, Args &&...args) {
  static int allowed = 0;
  if (smem > allowed) {
    cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute(%d bytes): %s", name, smem, cudaGetErrorString(e));
      return 2;
    }
    allowed = smem;
  }
  launch_pdl(Kernel, dim3(grid), dim3(threads), smem, stream, std::forward<Args>(args)...);
  RAVE_CHECK_LAUNCH(name);
  return 0;
}

// ------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled from the driver the runtime uses (null if it has none)
static inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)ptr;
  }
  return fn;
}

// Tiled map of a bf16 tensor of `rank` dimensions (innermost first; strides in bytes of dimensions 1 ..), dense
// boxes, out-of-range elements zero-filled.  The caller has checked get_encode_fn().
static inline CUresult encode_bf16_map(CUtensorMap *m, int rank, const void *base, const cuuint64_t *dims,
                                       const cuuint64_t *strides, const cuuint32_t *box, CUtensorMapSwizzle swizzle,
                                       CUtensorMapL2promotion promo) {
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return get_encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void *>(base), dims, strides,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// ------------------------------------------------------------------ descriptors
// wgmma shared-memory matrix descriptor: start address, LBO, SBO (all >> 4), layout type in bits 62-63
// (1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B).  The swizzle is a function of the absolute shared-memory
// address (as TMA writes it), so a start address moved by whole rows or by 32 bytes inside a row stays valid.
__host__ __device__ constexpr uint64_t wgmma_layout_for_swizzle(int swizzle_bytes) {
  return swizzle_bytes == 128 ? 1ull : (swizzle_bytes == 64 ? 2ull : (swizzle_bytes == 32 ? 3ull : 0ull));
}
// K-major operand tile whose rows are exactly one swizzle span wide: SBO = 8 rows * span, LBO unused
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr, int swizzle_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(((8u * (uint32_t)swizzle_bytes) >> 4) & 0x3FFF) << 32;  // stride byte offset
  d |= wgmma_layout_for_swizzle(swizzle_bytes) << 62;
  return d;
}
// MN-major operand (the reduction runs over tile ROWS, channels are contiguous): 64-channel slabs of 128-byte rows,
// SWIZZLE_128B; LBO = stride between 64-channel slabs, SBO = 8 rows
__device__ __forceinline__ uint64_t make_mnmajor_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;   // stride between 64-channel slabs
  d |= (uint64_t)((1024u >> 4) & 0x3FFF) << 32;        // stride between 8-row groups
  d |= 1ull << 62;                                     // SWIZZLE_128B
  return d;
}

}  // namespace tc
}  // namespace rave
