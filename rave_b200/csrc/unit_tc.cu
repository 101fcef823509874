// Fused Residual(DilatedUnit) forward on wgmma (sm_90a):
//
//     out = x + Conv1x1( LeakyReLU( Conv3_dil( LeakyReLU(x) ) ) )            rave/blocks.py:31-45 (Residual), 83-112 (DilatedUnit)
//
// in ONE kernel.  The reference runs 2 cuDNN convs + 2 activations + pads + the add (7 kernels, 5 HBM round trips);
// the per-layer tensor-core path (conv_tc.cu) still needed 2 launches with the intermediate operand a1 = LeakyReLU(conv3)
// going through HBM.  Here a CTA owns a tile of 128 time steps x ALL C channels:
//
//   phase 1   acc[128 x NC] (registers of the MMA warpgroup) = sum_{tap k<3} sum_kb  A_k[128 x BK] (TMA, rows shifted by
//             k*dil - pad) * W3_k[NC x BK]^T
//   epilogue1 acc -> LeakyReLU -> bf16 -> shared memory, written directly in the K-major swizzled layout the tensor
//             core reads (the A operand of phase 2 never leaves the SM); optionally also to HBM (training keeps a1 for the
//             backward: write-only, no read)
//   phase 2   acc[128 x NC] = sum_kb  A2[128 x BK] (shared memory) * W1[NC x BK]^T
//   epilogue2 acc + skip -> out (bf16 operand of the next layer and / or the fp32 stream); the skip h = x is
//             recovered from the unit's own input operand a = LeakyReLU(x) (inverse LeakyReLU), as conv_tc.cu does
//
// The channels run in N chunks of NC = 96 (the accumulators of a 128 x NC chunk are NC registers per MMA thread); the
// 128 x C bf16 A2 tile stays resident (96 KB at C = 384).  A finished chunk goes to a shared-memory buffer that the
// epilogue reads while the warpgroup computes the next chunk -- except at the phase-1 -> phase-2 boundary of a tile,
// where phase 2 needs the complete A2.
// Algorithmic HBM bytes per unit: 2 B*L*C (operand in) + 2 B*L*C (operand out) [+ 2 B*L*C a1 when training] + 8 C^2
// (weights) -- C = 96, L = 4096, B = 32: 50 MB of HBM traffic instead of 126 MB for the two-launch form.
//
// Warp roles (416 threads): 0-3 = MMA warpgroup, 4 = TMA producer, 5..12 = epilogue (two warps per 32-row quarter of
// the tile, alternate 32-column chunks).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace rave {
namespace tc {

constexpr int U_THREADS = 416;
constexpr int U_EPI_WARPS = 8;
constexpr int U_SMEM_MAX = 227 * 1024;

struct UnitParams {
  int B, C, L, pitch;          // channel-last [B][pitch][C] operand tensors; L valid rows
  int dil, pad_l;
  int BL, BB, n_lt, n_bg;      // tile = BB batches x BL rows (BL * BB == 128)
  float slope_in_inv;          // 1 / slope of the LeakyReLU that produced the input operand (skip recovery)
  float slope_mid;             // LeakyReLU between the two convs
  int act_out;                 // activation applied to the written operand (RAVE_ACT_NONE / RAVE_ACT_LEAKY)
  float slope_out;
  const __nv_bfloat16 *xa;     // input operand (also the skip source)
  __nv_bfloat16 *a1_out;       // [B][pitch][C] or null: the intermediate operand, kept for the backward
  float *out_f32;              // [B][pitch][C] or null
  __nv_bfloat16 *out_act;      // [B][pitch][C] or null
};

template <int C, int BK>
struct UnitCfg {
  static constexpr int NC = 96;                               // N chunk: NC accumulator registers per MMA thread
  static constexpr int NCH = C / NC;
  static constexpr int KB = C / BK;                           // K blocks per tap
  static constexpr int SWZ = BK * 2;
  static constexpr int A_BYTES = 128 * BK * 2;
  static constexpr int B_BYTES = NC * BK * 2;
  static constexpr int B_PAD = (B_BYTES + 1023) / 1024 * 1024;
  static constexpr int STAGE_BYTES = A_BYTES + B_PAD;
  static constexpr int A2_SLAB = 128 * BK * 2;
  static constexpr int A2_BYTES = KB * A2_SLAB;               // the whole [128 x C] bf16 tile
  static constexpr int ACC_LD = acc_pitch(NC);
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;          // fp32 accumulator hand-over buffer
  static constexpr int MAX_STAGES = (U_SMEM_MAX - 256 - 1024 - A2_BYTES - ACC_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = MAX_STAGES > 6 ? 6 : MAX_STAGES;
  static constexpr int A2_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int ACC_OFFSET = A2_OFFSET + A2_BYTES;
  static constexpr int BAR_OFFSET = ACC_OFFSET + ACC_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;
  static_assert(STAGES >= 2, "not enough shared memory for a 2-stage pipeline");
  static_assert(NC % 32 == 0 && C % NC == 0, "chunk must be a multiple of 32 columns and tile C");
};

__device__ __forceinline__ float bfl(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bfh(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }

template <int C, int BK>
__global__ void __launch_bounds__(U_THREADS, 1)
dilated_unit_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w3,
                       const __grid_constant__ CUtensorMap tmap_w1, const UnitParams p) {
  using L = UnitCfg<C, BK>;
  constexpr int STAGES = L::STAGES, NC = L::NC, NCH = L::NCH, KB = L::KB, SWZ = L::SWZ;

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t *a2 = smem + L::A2_OFFSET;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::BAR_OFFSET);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *tfull_bar = empty_bar + STAGES;             // MMA -> epilogue: the accumulator buffer holds a chunk
  uint64_t *tempty_bar = tfull_bar + 1;                 // epilogue -> MMA: the buffer has been read
  uint64_t *a2_ready = tempty_bar + 1;                  // epilogue -> MMA: the tile's A2 operand is complete
  uint64_t *a2_free = a2_ready + 1;                     // MMA -> epilogue: phase 2 has finished reading A2

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w3);
    tma_prefetch_desc(&tmap_w1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);                      // one arrival per MMA warp
    }
    mbar_init(tfull_bar, 128);
    mbar_init(tempty_bar, U_EPI_WARPS);
    mbar_init(a2_ready, U_EPI_WARPS);
    mbar_init(a2_free, 4);
    fence_barrier_init();
    acc_bind(smem + L::ACC_OFFSET, L::ACC_LD);
  }
  __syncthreads();
  griddep_launch_dependents();      // dependents may begin their prologue ...
  griddep_wait();                   // ... and this kernel touches global memory only after its predecessors are done

  if (warp == 4) {
    // =========================== TMA producer ===========================
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int lt = tile % p.n_lt, bg = tile / p.n_lt;
      const int l0 = lt * p.BL, b0 = bg * p.BB;
      for (int ch = 0; ch < NCH; ++ch) {                 // phase 1: activation rows + conv3 weights
        for (int k = 0; k < 3; ++k) {
          const int row = l0 + k * p.dil - p.pad_l;
          for (int kb = 0; kb < KB; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t *sa = smem + stage * L::STAGE_BYTES;
            if (elect_one()) {
              mbar_arrive_expect_tx(&full_bar[stage], L::A_BYTES + L::B_BYTES);
              tma_load_4d(sa, &tmap_a, &full_bar[stage], kb * BK, 0, row, b0);
              tma_load_2d(sa + L::A_BYTES, &tmap_w3, &full_bar[stage], kb * BK, k * C + ch * NC);
            }
            __syncwarp();
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
      for (int ch = 0; ch < NCH; ++ch) {                 // phase 2: conv1 weights only (A2 is resident)
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t *sa = smem + stage * L::STAGE_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[stage], L::B_BYTES);
            tma_load_2d(sa + L::A_BYTES, &tmap_w1, &full_bar[stage], kb * BK, ch * NC);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < 4) {
    // =========================== MMA warpgroup ===========================
    constexpr uint64_t A_HALF = (64 * SWZ) >> 4;         // rows 64 .. 127 of a K-major operand tile
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t a2_base = smem_u32(a2);
    float d[2][NC / 2];
    int stage = 0;
    uint32_t phase = 0;
    int job = 0, it = 0;
    // hand a finished chunk to the epilogue once it has read the previous one
    auto hand_over = [&]() {
      mbar_wait(tempty_bar, (job & 1) ^ 1);
      acc_store<NC>(d, threadIdx.x);
      mbar_arrive(tfull_bar);
      ++job;
    };
    auto release = [&](bool free_a2) {
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<NC / 2>(d[0]);
      wgmma_fence_regs<NC / 2>(d[1]);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[stage]);
        if (free_a2) mbar_arrive(a2_free);               // this warp's MMAs no longer read A2
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      for (int ch = 0; ch < NCH; ++ch) {                 // ---- phase 1
        for (int u = 0; u < 3 * KB; ++u) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_base + stage * L::STAGE_BYTES;
          const uint64_t adesc = make_kmajor_desc(sa, SWZ);
          const uint64_t bdesc = make_kmajor_desc(sa + L::A_BYTES, SWZ);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
              Wgmma<NC, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc + 2 * kk, (u > 0 || kk > 0) ? 1u : 0u);
          }
          release(false);
        }
        hand_over();
      }
      mbar_wait(a2_ready, it & 1);                       // every epilogue warp has written (and fenced) its A2 rows
      for (int ch = 0; ch < NCH; ++ch) {                 // ---- phase 2
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sb = smem_base + stage * L::STAGE_BYTES + L::A_BYTES;
          const uint64_t adesc = make_kmajor_desc(a2_base + kb * L::A2_SLAB, SWZ);
          const uint64_t bdesc = make_kmajor_desc(sb, SWZ);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
              Wgmma<NC, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc + 2 * kk, (kb > 0 || kk > 0) ? 1u : 0u);
          }
          release(ch == NCH - 1 && kb == KB - 1);
        }
        hand_over();
      }
    }
  } else {
    // =========================== epilogue (8 warps) ===========================
    const int quad = warp & 3;                           // rows quad * 32 .. quad * 32 + 31 of the tile
    const int part = (warp - 5) >> 2;                    // 0 / 1: alternate 32-column chunks
    const int row = quad * 32 + lane;
    // byte offset of this row's 16-byte chunk c16 inside an A2 slab: row * SWZ + ((c16 ^ swz(row)) << 4)
    const uint32_t row_xor = (SWZ == 128) ? (uint32_t)(row & 7) : (SWZ == 64) ? (uint32_t)((row >> 1) & 3)
                                                                                : (uint32_t)((row >> 2) & 1);
    int job = 0, it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int lt = tile % p.n_lt, bg = tile / p.n_lt;
      const int b = bg * p.BB + row / p.BL;
      const int l = lt * p.BL + row % p.BL;
      const bool valid = (b < p.B) && (l < p.L);
      const size_t grow = ((size_t)b * p.pitch + l) * C;
      if (it > 0) mbar_wait(a2_free, (it - 1) & 1);      // the previous tile's phase 2 no longer reads A2
      // ---- epilogue 1: acc -> LeakyReLU -> bf16 -> A2 (swizzled K-major rows) [+ HBM copy for the backward]
      for (int ch = 0; ch < NCH; ++ch, ++job) {
        mbar_wait(tfull_bar, job & 1);
        const uint32_t taddr = (uint32_t)(quad * 32) << 16;
#pragma unroll 1
        for (int c0 = part * 32; c0 < NC; c0 += 64) {
          float v[32];
          tmem_ld_32x32(taddr + c0, v);
          uint32_t pk[16];
#pragma unroll
          for (int w = 0; w < 16; ++w) {
            const float a0 = fmaxf(v[2 * w], v[2 * w] * p.slope_mid), a1 = fmaxf(v[2 * w + 1], v[2 * w + 1] * p.slope_mid);
            __nv_bfloat162 h = __floats2bfloat162_rn(a0, a1);
            pk[w] = *reinterpret_cast<uint32_t *>(&h);
          }
          const int col = ch * NC + c0;                  // first channel of this 32-column chunk
#pragma unroll
          for (int q = 0; q < 4; ++q) {                  // four 16-byte pieces (8 channels each)
            const int cc = col + 8 * q;
            const uint32_t off = (uint32_t)(cc / BK) * L::A2_SLAB + (uint32_t)row * SWZ +
                                 ((((uint32_t)(cc % BK) >> 3) ^ row_xor) << 4);
            *reinterpret_cast<uint4 *>(a2 + off) = make_uint4(pk[4 * q], pk[4 * q + 1], pk[4 * q + 2], pk[4 * q + 3]);
          }
          if (p.a1_out && valid) {
            stg256(p.a1_out + grow + col, pk);
            stg256(p.a1_out + grow + col + 16, pk + 8);
          }
        }
        if (ch == NCH - 1) fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(tempty_bar);
          if (ch == NCH - 1) mbar_arrive(a2_ready);
        }
      }
      // ---- epilogue 2: acc + skip -> outputs
      for (int ch = 0; ch < NCH; ++ch, ++job) {
        // skip rows of this thread's chunks: issue the loads before waiting for the accumulator
        uint32_t sk[(NC + 63) / 64][16];
#pragma unroll
        for (int i = 0; i < (NC + 63) / 64; ++i) {
          const int c0 = part * 32 + 64 * i;
          if (c0 < NC && valid) {
            ldg256(p.xa + grow + ch * NC + c0, sk[i]);
            ldg256(p.xa + grow + ch * NC + c0 + 16, sk[i] + 8);
          }
        }
        mbar_wait(tfull_bar, job & 1);
        const uint32_t taddr = (uint32_t)(quad * 32) << 16;
#pragma unroll
        for (int i = 0; i < (NC + 63) / 64; ++i) {
          const int c0 = part * 32 + 64 * i;
          if (c0 < NC) {
            float v[32];
            tmem_ld_32x32(taddr + c0, v);
            if (valid) {
              const int col = ch * NC + c0;
#pragma unroll
              for (int w = 0; w < 16; ++w) {
                const float s0 = bfl(sk[i][w]), s1 = bfh(sk[i][w]);
                v[2 * w] += fminf(s0, s0 * p.slope_in_inv);          // inverse LeakyReLU of the input operand
                v[2 * w + 1] += fminf(s1, s1 * p.slope_in_inv);
              }
              if (p.out_f32) {
                uint32_t o[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) o[j] = __float_as_uint(v[j]);
#pragma unroll
                for (int j = 0; j < 4; ++j) stg256(p.out_f32 + grow + col + 8 * j, o + 8 * j);
              }
              if (p.out_act) {
                uint32_t pk[16];
#pragma unroll
                for (int w = 0; w < 16; ++w) {
                  float a0 = v[2 * w], a1 = v[2 * w + 1];
                  if (p.act_out == RAVE_ACT_LEAKY) {
                    a0 = fmaxf(a0, a0 * p.slope_out);
                    a1 = fmaxf(a1, a1 * p.slope_out);
                  }
                  __nv_bfloat162 h = __floats2bfloat162_rn(a0, a1);
                  pk[w] = *reinterpret_cast<uint32_t *>(&h);
                }
                stg256(p.out_act + grow + col, pk);
                stg256(p.out_act + grow + col + 16, pk + 8);
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(tempty_bar);
      }
    }
  }
}

// =============================================================================================
// Weight-stationary variant for the narrow units (C = 96: the six longest launches of the encoder / generator forward).
// dilated_unit_tc_kernel re-streams, for EVERY 128-row tile, the three tap-shifted copies of the activation rows
// (3 x 24 KB) and the whole weight set (W3 54 KB + W1 18 KB) from L2: 144 KB per tile.  Here the weights are loaded
// ONCE per CTA and stay in shared memory (72 KB), and each tile brings ONE haloed activation tile (128 + 2 dil rows):
// tap k is the same tile read (k dil) rows further down -- K-major operand, 64-byte swizzle, descriptor start address
// moved by whole rows (the swizzle is a function of the absolute shared-memory address, which is how TMA wrote it).
// 29 KB instead of 144 KB per tile.  The MMA warpgroup runs the epilogues itself, straight from its accumulator
// registers: the intermediate a1 goes into the swizzled A2 tile (the phase-2 A operand, and the source of its TMA store
// to HBM), the skip comes from the centre rows of the haloed tile, the bf16 output leaves through a staging tile and TMA.
// Warp roles (160 threads): 0-3 = MMA warpgroup + epilogues, 4 = TMA producer.
// =============================================================================================
constexpr int UW_THREADS = 160;
constexpr int UW_AROWS = 152;                       // 128 + 2 * dil rows, dil <= 12
constexpr int UW_ASLAB = UW_AROWS * 64;             // one 32-channel K block of the haloed tile (64-byte rows)
constexpr int UW_WSLAB = 96 * 64;                   // one (tap, K block) weight slab: 96 rows x 32 channels
constexpr int UW_STAGES = 3;
constexpr int UW_W3_OFF = 0, UW_W1_OFF = 9 * UW_WSLAB, UW_A_OFF = 12 * UW_WSLAB;
constexpr int UW_A2_OFF = UW_A_OFF + UW_STAGES * 3 * UW_ASLAB;
constexpr int UW_OUT_OFF = UW_A2_OFF + 3 * (128 * 64);      // staging tile of the bf16 output (TMA store source)
constexpr int UW_BAR_OFF = UW_OUT_OFF + 3 * (128 * 64);
constexpr int UW_TOTAL = UW_BAR_OFF + 256 + 1024;
static_assert(UW_TOTAL <= U_SMEM_MAX, "weight-stationary unit: shared memory");

// byte offset of channel c (even) of row `row` in a [rows][32 ch] 64-byte-swizzled K-block sequence of `slab` bytes
__device__ __forceinline__ uint32_t sw64_off(int row, int c, uint32_t slab) {
  return (uint32_t)(c >> 5) * slab + (uint32_t)row * 64u + ((((uint32_t)(c & 31) >> 3) ^ (((uint32_t)row >> 1) & 3u)) << 4) +
         (uint32_t)(c & 7) * 2u;
}

__global__ void __launch_bounds__(UW_THREADS, 1)
dilated_unit_ws96_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w3,
                         const __grid_constant__ CUtensorMap tmap_w1, const __grid_constant__ CUtensorMap tmap_out,
                         const __grid_constant__ CUtensorMap tmap_a1, const UnitParams p) {
  constexpr int C = 96, BK = 32, KB = 3, SWZ = 64, A2_SLAB = 128 * 64;
  constexpr uint64_t A_HALF = (64 * SWZ) >> 4;        // rows 64 .. 127 of a K-major operand tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t *a2 = smem + UW_A2_OFF;
  uint8_t *outb = smem + UW_OUT_OFF;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + UW_BAR_OFF);
  uint64_t *empty_bar = full_bar + UW_STAGES;
  uint64_t *w_bar = empty_bar + UW_STAGES;              // the resident weights have landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w3);
    tma_prefetch_desc(&tmap_w1);
    for (int s = 0; s < UW_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);      // released by the MMA warps once the epilogue has read the skip rows
    }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();
  griddep_wait();
  const int arows = 128 + 2 * p.dil;                    // rows of the haloed tile actually loaded

  if (warp == 4) {
    // =========================== TMA producer ===========================
    if (elect_one()) {                                   // weights: once
      mbar_arrive_expect_tx(w_bar, 12 * UW_WSLAB);
      for (int k = 0; k < 3; ++k)
        for (int kb = 0; kb < KB; ++kb)
          tma_load_2d(smem + UW_W3_OFF + (k * KB + kb) * UW_WSLAB, &tmap_w3, w_bar, kb * BK, k * C);
      for (int kb = 0; kb < KB; ++kb) tma_load_2d(smem + UW_W1_OFF + kb * UW_WSLAB, &tmap_w1, w_bar, kb * BK, 0);
    }
    __syncwarp();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int lt = tile % p.n_lt, b0 = tile / p.n_lt;          // BB == 1
      const int row0 = lt * 128 - p.pad_l;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      uint8_t *sa = smem + UW_A_OFF + stage * 3 * UW_ASLAB;
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(KB * arows * 64));
        for (int kb = 0; kb < KB; ++kb) tma_load_4d(sa + kb * UW_ASLAB, &tmap_a, &full_bar[stage], kb * BK, 0, row0, b0);
      }
      __syncwarp();
      if (++stage == UW_STAGES) { stage = 0; phase ^= 1; }
    }
    return;
  }
  // =========================== MMA warpgroup + epilogues ===========================
  // fragment of this thread (see acc_store): rows r0 + 8 e + 64 h, columns 8 j + 2 (lane % 4) + {0, 1}
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  const bool issuer = threadIdx.x == 0;
  const uint32_t smem_base = smem_u32(smem);
  float d[2][C / 2];
  mbar_wait(w_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int lt = tile % p.n_lt, b = tile / p.n_lt;
    const int l0 = lt * 128;
    // ---- phase 1: conv3 over the haloed tile
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_base + UW_A_OFF + stage * 3 * UW_ASLAB;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const uint64_t adesc = make_kmajor_desc(sa + kb * UW_ASLAB + (uint32_t)(k * p.dil) * 64u, SWZ);
        const uint64_t bdesc = make_kmajor_desc(smem_base + UW_W3_OFF + (k * KB + kb) * UW_WSLAB, SWZ);
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            Wgmma<C, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc + 2 * kk, (k > 0 || kb > 0 || kk > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<C / 2>(d[0]);
    wgmma_fence_regs<C / 2>(d[1]);
    // ---- epilogue 1: LeakyReLU -> bf16 -> A2 (swizzled K-major rows).  The previous tile's phase 2 has retired (same
    // warpgroup); its a1 store must be done reading A2 (bulk groups complete in order: a1, out, a1, out ...)
    if (p.a1_out && issuer) {
      if (p.out_act) bulk_wait_read<1>();
      else bulk_wait_read<0>();
    }
    named_bar_sync(1, 128);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int row = 64 * h + r0 + 8 * e;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const float v0 = d[h][4 * j + 2 * e], v1 = d[h][4 * j + 2 * e + 1];
          const __nv_bfloat162 a = __floats2bfloat162_rn(fmaxf(v0, v0 * p.slope_mid), fmaxf(v1, v1 * p.slope_mid));
          *reinterpret_cast<__nv_bfloat162 *>(a2 + sw64_off(row, 8 * j + cq, A2_SLAB)) = a;
        }
      }
    fence_proxy_async();                                  // generic-proxy smem writes -> tensor core / TMA
    named_bar_sync(1, 128);
    if (p.a1_out && issuer) {                             // training: keep a1 for the backward (write-only)
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) tma_store_4d(&tmap_a1, a2 + kb * A2_SLAB, kb * BK, 0, l0, b);
      bulk_commit();
    }
    // ---- phase 2: 1x1 conv on the resident A2 / W1
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const uint64_t adesc = make_kmajor_desc(smem_base + UW_A2_OFF + kb * A2_SLAB, SWZ);
      const uint64_t bdesc = make_kmajor_desc(smem_base + UW_W1_OFF + kb * UW_WSLAB, SWZ);
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          Wgmma<C, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc + 2 * kk, (kb > 0 || kk > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<C / 2>(d[0]);
    wgmma_fence_regs<C / 2>(d[1]);
    // ---- epilogue 2: acc + skip (centre rows of the haloed tile) -> outputs
    if (p.out_act && issuer) {                            // the previous tile's output store has read `outb`
      if (p.a1_out) bulk_wait_read<1>();                  // ... this tile's a1 store may still be running
      else bulk_wait_read<0>();
    }
    if (p.out_act) named_bar_sync(1, 128);
    const uint8_t *sah = smem + UW_A_OFF + stage * 3 * UW_ASLAB;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int row = 64 * h + r0 + 8 * e;
        const int l = l0 + row;
        const bool valid = l < p.L;
        const size_t grow = ((size_t)b * p.pitch + l) * C;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int c = 8 * j + cq;
          const __nv_bfloat162 sk = *reinterpret_cast<const __nv_bfloat162 *>(sah + sw64_off(row + p.pad_l, c, UW_ASLAB));
          const float s0 = __low2float(sk), s1 = __high2float(sk);
          float v0 = d[h][4 * j + 2 * e] + fminf(s0, s0 * p.slope_in_inv);     // inverse LeakyReLU of the input
          float v1 = d[h][4 * j + 2 * e + 1] + fminf(s1, s1 * p.slope_in_inv);
          if (p.out_f32 && valid) *reinterpret_cast<float2 *>(p.out_f32 + grow + c) = make_float2(v0, v1);
          if (p.out_act) {
            if (p.act_out == RAVE_ACT_LEAKY) {
              v0 = fmaxf(v0, v0 * p.slope_out);
              v1 = fmaxf(v1, v1 * p.slope_out);
            }
            *reinterpret_cast<__nv_bfloat162 *>(outb + sw64_off(row, c, A2_SLAB)) = __floats2bfloat162_rn(v0, v1);
          }
        }
      }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);      // skip rows read: the producer may refill this stage
    if (p.out_act) {
      fence_proxy_async();
      named_bar_sync(1, 128);
      if (issuer) {
#pragma unroll
        for (int kb = 0; kb < KB; ++kb) tma_store_4d(&tmap_out, outb + kb * A2_SLAB, kb * BK, 0, l0, b);
        bulk_commit();
      }
    }
    if (++stage == UW_STAGES) { stage = 0; phase ^= 1; }
  }
  if (issuer) bulk_wait_all();
}

typedef CUresult (*EncodeTiledFnU)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                   const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFnU unit_encode_fn() {
  static EncodeTiledFnU fn = nullptr;
  if (!fn) {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFnU)ptr;
  }
  return fn;
}

template <int C, int BK>
static int launch_unit(const CUtensorMap &ta, const CUtensorMap &t3, const CUtensorMap &t1, const UnitParams &p,
                       cudaStream_t stream) {
  using L = UnitCfg<C, BK>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dilated_unit_tc_kernel<C, BK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         L::TOTAL);
    if (e != cudaSuccess) {
      set_error("dilated_unit_tc: cudaFuncSetAttribute(%d bytes): %s", L::TOTAL, cudaGetErrorString(e));
      return 2;
    }
    attr = true;
  }
  const int tiles = p.n_lt * p.n_bg;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = tiles < sms ? tiles : sms;
  launch_pdl(dilated_unit_tc_kernel<C, BK>, dim3(grid), dim3(U_THREADS), L::TOTAL, stream, ta, t3, t1, p);
  RAVE_CHECK_LAUNCH("dilated_unit_tc");
  return 0;
}

}  // namespace tc
}  // namespace rave

extern "C" int rave_dilated_unit_tc_supported(int C, int L) {
  return (C == 96 || C == 192 || C == 384) && L >= 8;
}

extern "C" int rave_dilated_unit_tc_fwd(const void *xa, const void *w3t, const void *w1t, void *a1_out, float *out_f32,
                                        void *out_act, int B, int C, int L, int pitch, int dil, int pad_l,
                                        float slope_in, float slope_mid, int act_out, float slope_out, void *stream) {
  using namespace rave;
  using namespace rave::tc;
  RAVE_CHECK_ARG(xa && w3t && w1t && (out_f32 || out_act), "dilated_unit_tc: null pointer");
  RAVE_CHECK_ARG(rave_dilated_unit_tc_supported(C, L), "dilated_unit_tc: unsupported width C=%d (96, 192, 384)", C);
  RAVE_CHECK_ARG(B > 0 && L > 0 && dil >= 1 && pad_l >= 0, "dilated_unit_tc: bad shape");
  if (pitch <= 0) pitch = L;
  RAVE_CHECK_ARG(pitch >= L, "dilated_unit_tc: pitch %d < L %d", pitch, L);
  RAVE_CHECK_ARG(slope_in > 0.f && slope_in <= 1.f && slope_mid >= 0.f && slope_mid <= 1.f && slope_out >= 0.f &&
                     slope_out <= 1.f, "dilated_unit_tc: LeakyReLU slopes must lie in (0, 1]");
  RAVE_CHECK_ARG(act_out == RAVE_ACT_NONE || act_out == RAVE_ACT_LEAKY, "dilated_unit_tc: output activation %d", act_out);
  RAVE_CHECK_ARG((((uintptr_t)xa | (uintptr_t)a1_out | (uintptr_t)out_f32 | (uintptr_t)out_act) & 31) == 0 &&
                     (((uintptr_t)w3t | (uintptr_t)w1t) & 15) == 0, "dilated_unit_tc: tensors must be 32-byte aligned");
  EncodeTiledFnU enc = unit_encode_fn();
  RAVE_CHECK_ARG(enc, "dilated_unit_tc: cuTensorMapEncodeTiled not available");
  const int BK = C % 64 == 0 ? 64 : 32;
  UnitParams p;
  p.B = B; p.C = C; p.L = L; p.pitch = pitch; p.dil = dil; p.pad_l = pad_l;
  int BL = 128;
  while (BL > L && BL > 8) BL >>= 1;
  p.BL = BL; p.BB = 128 / BL;
  p.n_lt = ceil_div(L, BL);
  p.n_bg = ceil_div(B, p.BB);
  p.slope_in_inv = 1.f / slope_in;
  p.slope_mid = slope_mid;
  p.act_out = act_out;
  p.slope_out = slope_out;
  p.xa = (const __nv_bfloat16 *)xa;
  p.a1_out = (__nv_bfloat16 *)a1_out;
  p.out_f32 = out_f32;
  p.out_act = (__nv_bfloat16 *)out_act;
  const CUtensorMapSwizzle swz = BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  const CUtensorMapL2promotion promo = BK == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  const int NC = 96;
  CUtensorMap ta, t3, t1;
  {
    cuuint64_t dims[4] = {(cuuint64_t)C, 1, (cuuint64_t)L, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2, (cuuint64_t)C * 2 * pitch};
    cuuint32_t box[4] = {(cuuint32_t)BK, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&ta, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(xa), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "dilated_unit_tc: tensor map A encode failed (%d)", (int)r);
  }
  for (int which = 0; which < 2; ++which) {
    cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)(which == 0 ? 3 : 1) * C};
    cuuint64_t strides[1] = {(cuuint64_t)C * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)NC};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(which == 0 ? &t3 : &t1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                     const_cast<void *>(which == 0 ? w3t : w1t), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swz, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "dilated_unit_tc: weight tensor map encode failed (%d)", (int)r);
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (C == 96 && p.BB == 1 && dil <= 12) {
    // weight-stationary kernel: its activation map carries the haloed box (128 + 2 dil rows), its weight maps one
    // (tap, K block) slab per box
    CUtensorMap tah, t3s, t1s;
    {
      cuuint64_t dims[4] = {(cuuint64_t)C, 1, (cuuint64_t)L, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2, (cuuint64_t)C * 2 * pitch};
      cuuint32_t box[4] = {32, 1, (cuuint32_t)(128 + 2 * dil), 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(&tah, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(xa), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      RAVE_CHECK_ARG(r == CUDA_SUCCESS, "dilated_unit_tc(ws): tensor map A encode failed (%d)", (int)r);
    }
    for (int which = 0; which < 2; ++which) {
      cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)(which == 0 ? 3 : 1) * C};
      cuuint64_t strides[1] = {(cuuint64_t)C * 2};
      cuuint32_t box[2] = {32, 96};
      cuuint32_t estr[2] = {1, 1};
      CUresult r = enc(which == 0 ? &t3s : &t1s, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                       const_cast<void *>(which == 0 ? w3t : w1t), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      RAVE_CHECK_ARG(r == CUDA_SUCCESS, "dilated_unit_tc(ws): weight tensor map encode failed (%d)", (int)r);
    }
    static bool attr = false;
    if (!attr) {
      cudaError_t er = cudaFuncSetAttribute(dilated_unit_ws96_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, UW_TOTAL);
      if (er != cudaSuccess) {
        set_error("dilated_unit_tc(ws): cudaFuncSetAttribute(%d bytes): %s", UW_TOTAL, cudaGetErrorString(er));
        return 2;
      }
      attr = true;
    }
    const int tiles = p.n_lt * p.n_bg;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // bf16 outputs leave through TMA: [B][pitch][96] viewed as (c, 1, row, b) boxes of one 32-channel K block x 128 rows
    // (rows >= L and batches >= B are clipped by the TMA unit)
    CUtensorMap tout, ta1;
    memset(&tout, 0, sizeof(tout));
    memset(&ta1, 0, sizeof(ta1));
    for (int which = 0; which < 2; ++which) {
      void *base = which == 0 ? out_act : a1_out;
      if (!base) continue;
      cuuint64_t dims[4] = {(cuuint64_t)C, 1, (cuuint64_t)L, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2, (cuuint64_t)C * 2 * pitch};
      cuuint32_t box[4] = {32, 1, 128, 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(which == 0 ? &tout : &ta1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      RAVE_CHECK_ARG(r == CUDA_SUCCESS, "dilated_unit_tc(ws): output tensor map encode failed (%d)", (int)r);
    }
    launch_pdl(dilated_unit_ws96_kernel, dim3(tiles < sms ? tiles : sms), dim3(UW_THREADS), UW_TOTAL, s, tah, t3s, t1s,
               tout, ta1, p);
    RAVE_CHECK_LAUNCH("dilated_unit_tc(ws)");
    return 0;
  }
  switch (C) {
    case 96: return launch_unit<96, 32>(ta, t3, t1, p, s);
    case 192: return launch_unit<192, 64>(ta, t3, t1, p, s);
    case 384: return launch_unit<384, 64>(ta, t3, t1, p, s);
  }
  set_error("dilated_unit_tc: no kernel for C=%d", C);
  return 1;
}
