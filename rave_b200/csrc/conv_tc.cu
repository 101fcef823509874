// wgmma conv1d engine (sm_90a): im2col-free implicit GEMM with the TIME axis on the MMA M dimension.
//
//   D[m = (b,l)][n = co] = sum_{tap k} sum_{ci}  A_k[(b,l)][ci] * W_k[co][ci]
//   A_k[(b,l)][ci] = xa[b][l*stride + k*dil - pad_l][ci]            (zero outside [0, Lin))
//
// Activations are CHANNEL-LAST bf16 (xa[b][l][c]): a tap shift / stride / dilation is then a pure ROW
// offset of a K-major operand tile, which TMA expresses with a 4-D tensor map (c, phase, l/stride, b)
// -- out-of-range rows (the conv padding) are zero-filled by the TMA unit, so there is no F.pad and no
// im2col buffer.  Weights are tap-major bf16 wt[k][co][ci] (K-major B operand).  Both operand tiles use
// the canonical K-major swizzled layout (row = one swizzle span = BLOCK_K*2 bytes).  One warpgroup issues the
// wgmma of a 128-row tile (two m64 halves) and keeps the accumulators in registers; a finished tile goes to a
// shared-memory buffer from which the epilogue (bias, residual, dual write of the pre-activation fp32 stream and the
// bf16 activated operand of the NEXT conv) reads it row by row while the warpgroup already runs the next tile.
// Warp roles: 0-3 = MMA warpgroup, 4 = TMA producer, 5-8 = epilogue.
//
// Replaces: cc.Conv1d.forward = F.pad + F.conv1d -> cuDNN (reference call sites rave/blocks.py:96-108,
// 538-592, 637-692; rave/discriminator.py:99-111), the preceding activation module and the residual add.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace rave {
namespace tc {

constexpr int BLOCK_M = 128;
constexpr int NUM_THREADS = 288;       // MMA warpgroup, producer warp, 4 epilogue warps
constexpr int SMEM_MAX = 227 * 1024;   // dynamic shared memory a CTA may opt into on sm_90

struct TcParams {
  int B, Cin, Lin, Cout, Lout, K, stride, dil, pad_l;
  int BL, BB;              // rows of one M tile: BB batches x BL time steps (BL*BB == 128)
  int n_lt, n_bg, n_nt;    // tile counts: time tiles, batch groups, N tiles
  int num_kb;              // K blocks per tap = ceil(Cin / BLOCK_K)
  int act;
  float slope;
  const float *bias;       // [Cout] or null
  const float *res;        // channel-last fp32 [B][out_rows][Cout] or null
  const __nv_bfloat16 *res_bf16;   // same, bf16 (gradient stream) or null
  const __nv_bfloat16 *dact_src;   // channel-last bf16 [B][out_rows][Cout] or null: out *= leaky'(dact_src)
  const __nv_bfloat16 *res_act;    // channel-last bf16 a = LeakyReLU(h) or null: out += h recovered from a
  float res_inv_slope;             //   (residual skip without a separate fp32 stream: h = a > 0 ? a : a / slope)
  float *out_f32;          // channel-last fp32 or null
  __nv_bfloat16 *out_act;  // channel-last bf16 = act(out) or null
  int out_rows;            // rows per batch of the output tensors (>= Lout when phases interleave)
  int out_row_stride;      // output row = l * out_row_stride + out_row_offset (transposed-conv phases)
  int out_row_offset;
  const float *fm_d;       // feature-matching gradient fused into a dgrad epilogue (or null): dact_src is the bf16
  long fm_half;            //   operand a = LeakyReLU(h) of [real; fake] rows, fm_half elements apart; adds
  int fm_bh;               //   d0 sgn(h_r-h_f) + d1 sgn(h_r) to real rows (b < fm_bh), -d0 sgn(h_r-h_f) to fake rows
  int x3;                  // split-operand mode ("bf16x3"): activations [.., 2*Cin] = [hi | lo], weights [2][K][Cout][Cin]
  int act_ld;              // row length (elements) of the bf16 operand tensors the epilogue touches (out_act, res_act):
                           // Cout, or 2*Cout in x3 mode
  int act_cs;              // x3: channels per POSITION of an output row (Cout; Cout/stride when the row holds the phases
                           // of a transposed conv side by side): column n = q*cs + c lives at q*2cs + c (hi), +cs (lo)
};

template <int BLOCK_N, int BLOCK_K, bool X3 = false>
struct SmemLayout {
  static constexpr int PARTS = X3 ? 2 : 1;                    // x3: hi and lo operand tiles side by side
  static constexpr int A_PART = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_PART = (BLOCK_N * BLOCK_K * 2 + 1023) / 1024 * 1024;
  static constexpr int A_BYTES = PARTS * A_PART;
  static constexpr int B_BYTES = PARTS * BLOCK_N * BLOCK_K * 2;          // bytes the TMA unit delivers
  static constexpr int B_BYTES_PAD = PARTS * B_PART;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES_PAD;
  static constexpr int ACC_LD = acc_pitch(BLOCK_N);
  static constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;                 // fp32 accumulator hand-over buffer
  static constexpr int MAX_STAGES = (SMEM_MAX - ACC_BYTES - 256 - 1024) / STAGE_BYTES;
  static constexpr int STAGES = MAX_STAGES > 8 ? 8 : MAX_STAGES;
  static constexpr int ACC_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = ACC_OFFSET + ACC_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;  // + barriers + alignment slack
  static_assert(STAGES >= 2, "not enough shared memory for a 2-stage pipeline");
};

// Epilogue of one 128 x BLOCK_N accumulator tile: this thread owns row (taddr >> 16) + lane of the accumulator buffer.
// One chunk = CW (16 or 32) consecutive channels.  All global loads of the chunk (residual, gradient skip,
// LeakyReLU' mask, feature-matching partner row) are issued BEFORE the accumulator load so that their latency overlaps it.
// Row segments move as whole 32-byte sectors per lane (two 128-bit accesses each).
template <int NWORDS>
__device__ __forceinline__ void ld_words(const void *ptr, uint32_t *w) {
  static_assert(NWORDS % 8 == 0, "256-bit granules");
#pragma unroll
  for (int i = 0; i < NWORDS / 8; ++i) ldg256(reinterpret_cast<const uint8_t *>(ptr) + 32 * i, w + 8 * i);
}
template <int NWORDS>
__device__ __forceinline__ void st_words(void *ptr, const uint32_t *w) {
  static_assert(NWORDS % 8 == 0, "256-bit granules");
#pragma unroll
  for (int i = 0; i < NWORDS / 8; ++i) stg256(reinterpret_cast<uint8_t *>(ptr) + 32 * i, w + 8 * i);
}
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }

template <int CW, bool X3>
__device__ __forceinline__ void tc_epi_chunk(const TcParams &p, uint32_t taddr, int co, bool valid, size_t orow,
                                             int fm_side = 0) {
  constexpr int NW = CW / 2;      // 32-bit words of a bf16 row segment
  float v[CW];
  uint32_t rf[CW], rb[NW], dm[NW], ra[NW], ra2[X3 ? NW : 1], pm[NW];
  const size_t off = orow * p.Cout + co;
  // bf16 operand tensors: in x3 mode every position is [hi | lo] (2 * act_cs channels)
  const int cs = X3 ? p.act_cs : 0;
  const size_t offa = X3 ? orow * (size_t)p.act_ld + (size_t)(co / cs) * (2 * cs) + (co % cs) : off;
  if (valid) {
    if (!X3 && fm_side)       // partner row of the other batch half (same position, same channels)
      ld_words<NW>(p.dact_src + (fm_side > 0 ? off + p.fm_half : off - p.fm_half), pm);
    if (p.res_act) {
      ld_words<NW>(p.res_act + offa, ra);
      if (X3) ld_words<NW>(p.res_act + offa + cs, ra2);
    }
    if (p.res) ld_words<CW>(p.res + off, rf);
    if (!X3 && p.res_bf16) ld_words<NW>(p.res_bf16 + off, rb);
    if (!X3 && p.dact_src) ld_words<NW>(p.dact_src + off, dm);
  }
  if (CW == 32) tmem_ld_32x32(taddr, v);
  else tmem_ld_32x16(taddr, v);
  if (!valid) return;
  if (p.bias) {
    const float4 *b4 = reinterpret_cast<const float4 *>(p.bias + co);
#pragma unroll
    for (int i = 0; i < CW / 4; ++i) {
      const float4 bb = __ldg(b4 + i);
      v[4 * i] += bb.x; v[4 * i + 1] += bb.y; v[4 * i + 2] += bb.z; v[4 * i + 3] += bb.w;
    }
  }
  if (!X3 && p.dact_src) {   // chain rule through the LeakyReLU that produced this conv's operand (sign bits of bf16)
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      if (dm[w] & 0x00008000u) v[2 * w] *= p.slope;
      if (dm[w] & 0x80000000u) v[2 * w + 1] *= p.slope;
    }
  }
  if (!X3 && fm_side) {
    // Gradient of d0 * sum|h_r - h_f| + d1 * sum|h_r| with respect to h.  LeakyReLU is strictly increasing, so
    // sgn(h_r - h_f) = sgn(a_r - a_f) and sgn(h_r) = sgn(a_r): the saved operands are compared as they are.  With
    // t = sgn(a_self - a_partner) both halves get d0 * t (real: d0 sgn(h_r-h_f); fake: -d0 sgn(h_r-h_f) = d0 t), real
    // rows d1 sgn(a_self) on top.  The epilogue is issue-bound on these launches: ~6 instructions per element
    // instead of ~20 for the literal form.
    const float d0 = __ldg(p.fm_d), d1 = fm_side > 0 ? __ldg(p.fm_d + 1) : 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float as = h ? bf_hi(dm[w]) : bf_lo(dm[w]);
        const float ap = h ? bf_hi(pm[w]) : bf_lo(pm[w]);
        const float t = (as > ap ? 1.f : 0.f) - (as < ap ? 1.f : 0.f);
        const float sr = (as > 0.f ? 1.f : 0.f) - (as < 0.f ? 1.f : 0.f);
        v[2 * w + h] = fmaf(d1, sr, fmaf(d0, t, v[2 * w + h]));
      }
    }
  }
  if (!X3 && p.res_bf16) {
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      v[2 * w] += bf_lo(rb[w]);
      v[2 * w + 1] += bf_hi(rb[w]);
    }
  }
  if (p.res_act) {     // residual skip from the unit's own bf16 operand: undo the LeakyReLU
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      float a0 = bf_lo(ra[w]), a1 = bf_hi(ra[w]);
      if (X3) {          // operand = hi + lo (exact in fp32: two 8-bit significands)
        a0 += bf_lo(ra2[w]);
        a1 += bf_hi(ra2[w]);
      }
      v[2 * w] += fminf(a0, a0 * p.res_inv_slope);          // inverse LeakyReLU (1/slope >= 1): two instructions
      v[2 * w + 1] += fminf(a1, a1 * p.res_inv_slope);
    }
  }
  if (p.res) {
#pragma unroll
    for (int i = 0; i < CW; ++i) v[i] += __uint_as_float(rf[i]);
  }
  if (p.out_f32) {
    uint32_t o[CW];
#pragma unroll
    for (int i = 0; i < CW; ++i) o[i] = __float_as_uint(v[i]);
    st_words<CW>(p.out_f32 + off, o);
  }
  if (p.out_act) {
    uint32_t pk[NW], pl[X3 ? NW : 1];
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      float a0 = v[2 * w], a1 = v[2 * w + 1];
      if (p.act == RAVE_ACT_LEAKY) {       // 0 <= slope <= 1 (checked on the host): max(x, slope x)
        a0 = fmaxf(a0, a0 * p.slope);
        a1 = fmaxf(a1, a1 * p.slope);
      }
      __nv_bfloat162 h = __floats2bfloat162_rn(a0, a1);
      pk[w] = *reinterpret_cast<uint32_t *>(&h);
      if (X3) {        // lo = bf16(a - hi): the operand is carried with a 16-bit significand
        __nv_bfloat162 l = __floats2bfloat162_rn(a0 - bf_lo(pk[w]), a1 - bf_hi(pk[w]));
        pl[w] = *reinterpret_cast<uint32_t *>(&l);
      }
    }
    st_words<NW>(p.out_act + offa, pk);
    if (X3) st_words<NW>(p.out_act + offa + cs, pl);
  }
}

template <int BLOCK_N, bool X3>
__device__ __forceinline__ void tc_epilogue(const TcParams &p, uint32_t taddr, int n0, bool valid, size_t orow,
                                            int fm_side) {
  constexpr int MAIN = BLOCK_N / 32 * 32;
  if (X3 && (p.act_cs & 31)) {
    // split-operand rows whose positions are 16 (mod 32) channels wide (capacity-48 transposed convs: 48 channels per
    // position): a 32-column chunk would straddle a [hi | lo] boundary -> 16-column chunks
#pragma unroll 1
    for (int c0 = 0; c0 < BLOCK_N; c0 += 16)
      tc_epi_chunk<16, X3>(p, taddr + c0, n0 + c0, valid, orow, fm_side);
    return;
  }
#pragma unroll 1
  for (int c0 = 0; c0 < MAIN; c0 += 32)
    tc_epi_chunk<32, X3>(p, taddr + c0, n0 + c0, valid, orow, fm_side);
  if (MAIN < BLOCK_N) tc_epi_chunk<16, X3>(p, taddr + MAIN, n0 + MAIN, valid, orow, fm_side);
}

template <int BLOCK_N, int BLOCK_K, bool X3>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const TcParams p) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  constexpr int STAGES = L::STAGES;
  constexpr int SWZ = BLOCK_K * 2;
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N >= 16 && BLOCK_N <= 128, "invalid wgmma N");

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::BAR_OFFSET);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *tfull_bar = empty_bar + STAGES;      // MMA warpgroup -> epilogue: the accumulator buffer holds a tile
  uint64_t *tempty_bar = tfull_bar + 1;          // epilogue -> MMA warpgroup: the buffer has been read

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg * p.n_nt;
  const int kblocks = p.K * p.num_kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);               // one arrival per MMA warp
    }
    mbar_init(tfull_bar, 128);
    mbar_init(tempty_bar, 4);
    fence_barrier_init();
    acc_bind(smem + L::ACC_OFFSET, L::ACC_LD);
  }
  __syncthreads();
  griddep_launch_dependents();      // dependents may begin their prologue ...
  griddep_wait();                   // ... and this kernel touches global memory only after its predecessors are done

  if (warp == 4) {
    // =========================== TMA producer (warp-uniform loop, elected lane issues) ===========================
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int nt = tile % p.n_nt;
      const int mt = tile / p.n_nt;
      const int lt = mt % p.n_lt;
      const int bg = mt / p.n_lt;
      const int l0 = lt * p.BL;
      const int b0 = bg * p.BB;
      const int n0 = nt * BLOCK_N;
      for (int k = 0; k < p.K; ++k) {
        // input row = l*stride + k*dil - pad_l = (l + j)*stride + ph
        const int off = k * p.dil - p.pad_l;
        int j = off / p.stride;
        int ph = off - j * p.stride;
        if (ph < 0) { ph += p.stride; j -= 1; }
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t *sa = smem + stage * L::STAGE_BYTES;
          uint8_t *sb = sa + L::A_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[stage], L::A_BYTES + L::B_BYTES);
            tma_load_4d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, ph, l0 + j, b0);
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, k * p.Cout + n0);
            if (X3) {      // lo halves: channels Cin.. of the activation rows, weight slabs K.. (wt is [2][K][Cout][Cin])
              tma_load_4d(sa + L::A_PART, &tmap_a, &full_bar[stage], p.Cin + kb * BLOCK_K, ph, l0 + j, b0);
              tma_load_2d(sb + L::B_PART, &tmap_b, &full_bar[stage], kb * BLOCK_K, (p.K + k) * p.Cout + n0);
            }
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < 4) {
    // =========================== MMA warpgroup ===========================
    // rows 64 h .. 64 h + 63 of an operand tile start 64 swizzle spans further: + (64 * SWZ) >> 4 in the address field
    constexpr uint64_t A_HALF = (64 * SWZ) >> 4;
    const uint32_t smem_base = smem_u32(smem);
    float d[2][BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_base + stage * L::STAGE_BYTES;
        const uint64_t adesc = make_kmajor_desc(sa, SWZ);
        const uint64_t bdesc = make_kmajor_desc(sa + L::A_BYTES, SWZ);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BLOCK_K / 16; ++kk) {
          // advance 16 bf16 = 32 bytes inside the swizzle span: +2 in the (addr >> 4) field
#pragma unroll
          for (int h = 0; h < 2; ++h)
            Wgmma<BLOCK_N, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc + 2 * kk, (kb > 0 || kk > 0) ? 1u : 0u);
        }
        if (X3) {        // a*w ~ a_hi*w_hi + a_lo*w_hi + a_hi*w_lo (the lo*lo term is below fp32 accumulation noise)
          const uint64_t adesc_lo = make_kmajor_desc(sa + L::A_PART, SWZ);
          const uint64_t bdesc_lo = make_kmajor_desc(sa + L::A_BYTES + L::B_PART, SWZ);
#pragma unroll
          for (int kk = 0; kk < BLOCK_K / 16; ++kk) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              Wgmma<BLOCK_N, 0, 0>::mma(d[h], adesc_lo + h * A_HALF + 2 * kk, bdesc + 2 * kk, 1u);
              Wgmma<BLOCK_N, 0, 0>::mma(d[h], adesc + h * A_HALF + 2 * kk, bdesc_lo + 2 * kk, 1u);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<BLOCK_N / 2>(d[0]);
        wgmma_fence_regs<BLOCK_N / 2>(d[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);           // this warp's MMAs no longer read the slot
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      mbar_wait(tempty_bar, (it & 1) ^ 1);                       // the epilogue has read the previous tile
      acc_store<BLOCK_N>(d, threadIdx.x);
      mbar_arrive(tfull_bar);
    }
  } else {
    // =========================== epilogue (4 warps) ===========================
    const int quad = warp & 3;           // rows quad * 32 .. quad * 32 + 31 of the tile
    const int row = quad * 32 + lane;    // row of the 128-row tile
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int nt = tile % p.n_nt;
      const int mt = tile / p.n_nt;
      const int lt = mt % p.n_lt;
      const int bg = mt / p.n_lt;
      const int n0 = nt * BLOCK_N;
      const int b = bg * p.BB + row / p.BL;
      const int l = lt * p.BL + row % p.BL;
      const bool valid = (b < p.B) && (l < p.Lout);
      const size_t orow = (size_t)b * p.out_rows + (size_t)l * p.out_row_stride + p.out_row_offset;

      mbar_wait(tfull_bar, it & 1);
      const uint32_t taddr = (uint32_t)(quad * 32) << 16;
      tc_epilogue<BLOCK_N, X3>(p, taddr, n0, valid, orow, p.fm_d ? (b < p.fm_bh ? 1 : -1) : 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
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

static CUtensorMapSwizzle swizzle_enum(int bytes) {
  return bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                 : CU_TENSOR_MAP_SWIZZLE_32B;
}

static int pick_block_k(int Cin) {
  if (Cin % 64 == 0) return 64;
  if (Cin % 32 == 0) return 32;
  if (Cin % 16 == 0) return 16;
  return 0;
}

static int pick_block_n(int Cout, long m_tiles) {
  // largest tile that still gives every SM work; Cout must be a multiple of it.  N <= 128: the MMA warpgroup holds the
  // 128 x N accumulator tile in registers (N fp32 per thread)
  const int cands[] = {128, 96, 64, 48, 32, 16};
  constexpr int NC = sizeof(cands) / sizeof(cands[0]);
  int best = 0;
  for (int c : cands) {
    if (Cout % c) continue;
    if (!best) best = c;
    if (m_tiles * (Cout / c) >= 132) return c;
  }
  // not enough tiles even at the smallest N: take the smallest valid one >= 32 if any
  for (int i = NC - 1; i >= 0; --i)
    if (Cout % cands[i] == 0 && cands[i] >= 32) return cands[i];
  return best;
}

template <int BN, int BK, bool X3>
static int launch(const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t stream) {
  using L = SmemLayout<BN, BK, X3>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, BK, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         L::TOTAL);
    if (e != cudaSuccess) {
      set_error("conv1d_tc: cudaFuncSetAttribute(%d bytes): %s", L::TOTAL, cudaGetErrorString(e));
      return 2;
    }
    attr = true;
  }
  const int tiles = p.n_lt * p.n_bg * p.n_nt;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = tiles < sms ? tiles : sms;
  launch_pdl(conv_tc_kernel<BN, BK, X3>, dim3(grid), dim3(NUM_THREADS), L::TOTAL, stream, ta, tb, p);
  RAVE_CHECK_LAUNCH("conv1d_tc");
  return 0;
}

template <int BK, bool X3>
static int dispatch_n(int bn, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p,
                      cudaStream_t s) {
  switch (bn) {
    case 128: return launch<128, BK, X3>(ta, tb, p, s);
    case 96: return launch<96, BK, X3>(ta, tb, p, s);
    case 64: return launch<64, BK, X3>(ta, tb, p, s);
    case 48: return launch<48, BK, X3>(ta, tb, p, s);
    case 32: return launch<32, BK, X3>(ta, tb, p, s);
    case 16: return launch<16, BK, X3>(ta, tb, p, s);
  }
  set_error("conv1d_tc: no kernel for BLOCK_N=%d", bn);
  return 1;
}

template <bool X3>
static int dispatch_all(int BK, int BN, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t s) {
  switch (BK) {
    case 64: return dispatch_n<64, X3>(BN, ta, tb, p, s);
    case 32: return dispatch_n<32, X3>(BN, ta, tb, p, s);
    case 16: return dispatch_n<16, X3>(BN, ta, tb, p, s);
  }
  set_error("conv1d_tc: no kernel for BLOCK_K=%d", BK);
  return 1;
}

// The split-operand (x3) instantiations live in their own translation unit (conv_tc_x3.cu includes this file with
// RAVE_TC_X3_UNIT defined) so that the two sets of kernels compile in parallel.
int conv_tc_dispatch_x3(int BK, int BN, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t s);
#ifdef RAVE_TC_X3_UNIT
int conv_tc_dispatch_x3(int BK, int BN, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t s) {
  return dispatch_all<true>(BK, BN, ta, tb, p, s);
}
#endif

}  // namespace tc
}  // namespace rave

#ifndef RAVE_TC_X3_UNIT
extern "C" int rave_conv1d_tc_supported(int Cin, int Cout, int K, int stride, int dil) {
  if (rave::tc::pick_block_k(Cin) == 0) return 0;
  if (Cout % 16) return 0;
  if (K < 1 || stride < 1 || dil < 1) return 0;
  return 1;
}

// Which kernel instance rave_conv1d_tc_fwd runs for a shape: BLOCK_N | BLOCK_K << 12; 0 = none.
extern "C" int rave_conv1d_tc_plan(int B, int Cin, int Cout, int Lout, int K) {
  using namespace rave;
  using namespace rave::tc;
  const int BK = pick_block_k(Cin);
  if (!BK || Cout % 16) return 0;
  int BL = 128;
  while (BL > Lout && BL > 8) BL >>= 1;
  const long m_tiles = (long)ceil_div(Lout, BL) * ceil_div(B, 128 / BL);
  const int BN = pick_block_n(Cout, m_tiles);
  if (!BN) return 0;
  return BN | (BK << 12);
}

static int conv1d_tc_fwd_impl(const void *xa, const void *wt, const float *bias, const float *res,
                              const void *res_bf16, const void *dact_src, const void *res_act, float res_slope,
                              float *out_f32, void *out_act,
                              int B, int Cin, int Lin, int in_pitch, int Cout, int Lout,
                              int K, int stride, int dil, int pad_l, int act, float slope, int out_rows,
                              int out_row_stride, int out_row_offset, const float *fm_d, int fm_bh,
                              void *stream, int x3, int act_cs = 0) {
  using namespace rave;
  using namespace rave::tc;
  RAVE_CHECK_ARG(!x3 || (!res_bf16 && !dact_src && !fm_d),
                 "conv1d_tc(x3): the split-operand mode has no gradient epilogues (forward path only)");
  RAVE_CHECK_ARG(xa && wt && (out_f32 || out_act), "conv1d_tc: null pointer");
  RAVE_CHECK_ARG(rave_conv1d_tc_supported(Cin, Cout, K, stride, dil), "conv1d_tc: unsupported shape Cin=%d Cout=%d",
                 Cin, Cout);
  if (in_pitch <= 0) in_pitch = Lin;
  RAVE_CHECK_ARG(in_pitch >= ceil_div(Lin, stride) * stride,
                 "conv1d_tc: input pitch %d < Lin %d rounded up to the stride %d (slack rows must be zero)", in_pitch,
                 Lin, stride);
  RAVE_CHECK_ARG(act == RAVE_ACT_NONE || act == RAVE_ACT_LEAKY, "conv1d_tc: epilogue activation %d unsupported", act);
  RAVE_CHECK_ARG(act != RAVE_ACT_LEAKY || (slope >= 0.f && slope <= 1.f), "conv1d_tc: LeakyReLU slope %g outside [0, 1]",
                 (double)slope);
  RAVE_CHECK_ARG(!res_act || (res_slope > 0.f && res_slope <= 1.f), "conv1d_tc: res_slope %g outside (0, 1]",
                 (double)res_slope);
  RAVE_CHECK_ARG(((uintptr_t)bias & 15) == 0, "conv1d_tc: bias must be 16-byte aligned");
  RAVE_CHECK_ARG(((uintptr_t)xa & 15) == 0 && ((uintptr_t)wt & 15) == 0, "conv1d_tc: operands must be 16B aligned");
  RAVE_CHECK_ARG((((uintptr_t)out_f32 | (uintptr_t)out_act | (uintptr_t)res | (uintptr_t)res_bf16 | (uintptr_t)dact_src |
                   (uintptr_t)res_act) & 31) == 0,
                 "conv1d_tc: epilogue tensors must be 32-byte aligned (256-bit row segments)");
  EncodeTiledFn enc = get_encode_fn();
  RAVE_CHECK_ARG(enc, "conv1d_tc: cuTensorMapEncodeTiled not available");

  const int BK = pick_block_k(Cin);
  // 256-byte L2 promotion over-fetches when a TMA row is a 64-byte (or shorter) span of a 192-byte channel row
  // (measured on the Cin = 96 layers: 209.6 -> 184.7 us); neutral to slightly positive for 128-byte spans.
  CUtensorMapL2promotion promo = BK == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  {
    const char *e = getenv("RAVE_TC_L2PROMO");
    if (e) promo = atoi(e) == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : atoi(e) == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                   : atoi(e) == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
  }
  TcParams p;
  p.B = B; p.Cin = Cin; p.Lin = Lin; p.Cout = Cout; p.Lout = Lout; p.K = K; p.stride = stride; p.dil = dil;
  p.pad_l = pad_l; p.act = act; p.slope = slope; p.bias = bias; p.res = res; p.out_f32 = out_f32;
  p.res_bf16 = (const __nv_bfloat16 *)res_bf16; p.dact_src = (const __nv_bfloat16 *)dact_src;
  p.res_act = (const __nv_bfloat16 *)res_act;
  p.res_inv_slope = (res_act && res_slope > 0.f) ? 1.f / res_slope : 1.f;
  p.out_act = (__nv_bfloat16 *)out_act;
  p.out_rows = out_rows > 0 ? out_rows : Lout;
  p.out_row_stride = out_row_stride > 0 ? out_row_stride : 1;
  p.out_row_offset = out_row_offset;
  RAVE_CHECK_ARG(!fm_d || (dact_src && slope > 0.f && ((fm_bh > 0 && 2 * fm_bh == B) || (fm_bh < 0 && -fm_bh == B))),
                 "conv1d_tc: the fused feature-matching gradient needs dact_src and a [real; fake] batch (B=%d, fm_bh=%d)",
                 B, fm_bh);
  p.fm_d = fm_d;
  p.fm_bh = fm_bh > 0 ? fm_bh : 0;                 // fm_bh < 0: every row is a fake row (partner |fm_bh| batches before)
  p.fm_half = (long)(fm_bh > 0 ? fm_bh : -fm_bh) * p.out_rows * Cout;
  p.x3 = x3 ? 1 : 0;
  p.act_ld = x3 ? 2 * Cout : Cout;
  p.act_cs = act_cs > 0 ? act_cs : Cout;
  RAVE_CHECK_ARG(!x3 || (Cout % p.act_cs == 0 && p.act_cs % 16 == 0),
                 "conv1d_tc(x3): %d channels per position do not tile the %d-column rows in 16-column chunks", p.act_cs,
                 Cout);
  RAVE_CHECK_ARG(!x3 || !res_act || p.act_cs == Cout, "conv1d_tc(x3): res_act needs one position per row");
  int BL = 128;
  while (BL > Lout && BL > 8) BL >>= 1;   // power of two <= max(Lout, 8)
  p.BL = BL; p.BB = 128 / BL;
  p.n_lt = ceil_div(Lout, BL);
  p.n_bg = ceil_div(B, p.BB);
  const int BN = pick_block_n(Cout, (long)p.n_lt * p.n_bg);
  RAVE_CHECK_ARG(BN > 0, "conv1d_tc: no BLOCK_N for Cout=%d", Cout);
  p.n_nt = Cout / BN;
  p.num_kb = ceil_div(Cin, BK);

  // A: channel-last activations viewed as (c, phase, l/stride, b)
  CUtensorMap ta, tb;
  {
    const cuuint64_t ca = (cuuint64_t)Cin * (x3 ? 2 : 1);       // channels per activation row ([hi | lo] in x3 mode)
    cuuint64_t dims[4] = {ca, (cuuint64_t)stride, (cuuint64_t)ceil_div(Lin, stride), (cuuint64_t)B};
    cuuint64_t strides[3] = {ca * 2, ca * 2 * stride, ca * 2 * in_pitch};
    cuuint32_t box[4] = {(cuuint32_t)BK, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&ta, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(xa), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(BK * 2), promo,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "conv1d_tc: tensor map A encode failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)Cin, (cuuint64_t)K * Cout * (x3 ? 2 : 1)};
    cuuint64_t strides[1] = {(cuuint64_t)Cin * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tb, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(wt), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(BK * 2), promo,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "conv1d_tc: tensor map B encode failed (%d)", (int)r);
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (x3) return conv_tc_dispatch_x3(BK, BN, ta, tb, p, s);
  return dispatch_all<false>(BK, BN, ta, tb, p, s);
}

extern "C" int rave_conv1d_tc_fwd(const void *xa, const void *wt, const float *bias, const float *res,
                                  const void *res_bf16, const void *dact_src, const void *res_act, float res_slope,
                                  float *out_f32, void *out_act,
                                  int B, int Cin, int Lin, int in_pitch, int Cout, int Lout,
                                  int K, int stride, int dil, int pad_l, int act, float slope, int out_rows,
                                  int out_row_stride, int out_row_offset, const float *fm_d, int fm_bh,
                                  void *stream) {
  return conv1d_tc_fwd_impl(xa, wt, bias, res, res_bf16, dact_src, res_act, res_slope, out_f32, out_act, B, Cin, Lin,
                            in_pitch, Cout, Lout, K, stride, dil, pad_l, act, slope, out_rows, out_row_stride,
                            out_row_offset, fm_d, fm_bh, stream, 0);
}

// Split-operand ("bf16x3") variant: the accurate fast mode.  xa: [B][in_pitch][2*Cin] bf16 rows [hi | lo] with
// x = hi + lo (16-bit significand), wt: [2][K][Cout][Cin] (all hi slabs, then all lo slabs); the tensor cores accumulate
// hi*hi + lo*hi + hi*lo in fp32 (relative error ~2^-17 per product instead of 2^-9).  out_act / res_act are [hi | lo]
// rows of 2*Cout; fp32 tensors as in rave_conv1d_tc_fwd.  act_cs (0 = Cout): channels per position when an output row
// holds several positions side by side (phase-fused transposed conv): each position is its own [hi | lo] pair.
// Forward only (no gradient epilogues).
extern "C" int rave_conv1d_tc_fwd_x3(const void *xa, const void *wt, const float *bias, const float *res,
                                     const void *res_act, float res_slope, float *out_f32, void *out_act,
                                     int B, int Cin, int Lin, int in_pitch, int Cout, int Lout,
                                     int K, int stride, int dil, int pad_l, int act, float slope, int out_rows,
                                     int out_row_stride, int out_row_offset, int act_cs, void *stream) {
  return conv1d_tc_fwd_impl(xa, wt, bias, res, nullptr, nullptr, res_act, res_slope, out_f32, out_act, B, Cin, Lin,
                            in_pitch, Cout, Lout, K, stride, dil, pad_l, act, slope, out_rows, out_row_stride,
                            out_row_offset, nullptr, 0, stream, 1, act_cs);
}

// =============================================================================================
// wgrad on wgmma:  dWt[k][m][n] += sum_{(b,l)} P[b][l][m] * Q[b][l*stride + k*dil - pad_l][n]
//
// P: channel-last bf16 [B][Lp][Cm] (conv: dy, M = Cout), Q: channel-last bf16 [B][Lq][Cn] (conv: the
// activated operand xa, N = Cin).  The reduction runs over tensor ROWS, so both operands are MN-major
// (the channel axis is contiguous): tiles are stored as 64-channel slabs [64 rows][64 ch] (128-byte
// rows, SWIZZLE_128B), LBO = slab stride, SBO = 8 rows.  One CTA owns one (m-tile, n-tile, tap) and one
// slice of the rows (split-K); partial tiles are combined with fp32 atomics into a pre-zeroed dWt.
// Reference: autograd of F.conv1d / F.conv_transpose1d (weight gradient) at the call sites listed above.
// =============================================================================================
namespace rave {
namespace tc {

constexpr int WG_ROWS = 64;             // reduction rows per pipeline stage
constexpr int WG_SLAB = WG_ROWS * 128;  // bytes of one [64 rows][64 ch] bf16 slab

struct WgParams {
  int B, Cm, Lp, Cn, Lq, K, stride, dil, pad_l;
  int BL, BB, n_lt, n_bg;   // row chunk = BB batches x BL rows (BL*BB == 64)
  int n_mt, n_nt, splits;
  float *dwt;               // [splits][K][Cm][Cn] fp32 partial sums (every element written exactly once)
  float *dbias;             // [Cm] pre-zeroed or null: += column sums of P (the bias gradient of a conv layer), formed
                            // by the tap-0 / n-tile-0 CTAs from the P tiles they stream anyway
  float *dbias_part;        // [splits][n_mt * 128] their per-slice partial sums (dbias_sum_kernel adds them up)
};

template <int BLOCK_N>
struct WgSmem {
  static constexpr int NS = (BLOCK_N + 63) / 64;
  static constexpr int STAGE_BYTES = (2 + NS) * WG_SLAB;
  static constexpr int MAX_STAGES = (200 * 1024) / STAGE_BYTES;
  static constexpr int STAGES = MAX_STAGES > 6 ? 6 : MAX_STAGES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int CS_OFFSET = BAR_OFFSET + 256;                 // column-sum scratch [8][128] fp32
  static constexpr int TOTAL = CS_OFFSET + 4096 + 1024;
};

template <int BLOCK_N>
__global__ void __launch_bounds__(NUM_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmap_p, const __grid_constant__ CUtensorMap tmap_q,
                const WgParams p) {
  using L = WgSmem<BLOCK_N>;
  constexpr int STAGES = L::STAGES;
  constexpr int NS = L::NS;
  static_assert(BLOCK_N % 64 == 0 && BLOCK_N <= 128, "MN-major B operand: whole 64-channel slabs");

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::BAR_OFFSET);
  uint64_t *empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // tile / slice owned by this CTA
  const int split = blockIdx.x % p.splits;
  int t = blockIdx.x / p.splits;
  const int nt = t % p.n_nt; t /= p.n_nt;
  const int mt = t % p.n_mt; t /= p.n_mt;
  const int k = t;
  const int m0 = mt * 128, n0 = nt * BLOCK_N;
  const int n_chunks = p.n_lt * p.n_bg;
  const int per = (n_chunks + p.splits - 1) / p.splits;
  const int ch_begin = split * per;
  const int ch_end = min(n_chunks, ch_begin + per);
  const int my_chunks = max(0, ch_end - ch_begin);
  const bool do_cs = p.dbias != nullptr && k == 0 && nt == 0;      // this CTA also reduces its P tiles over rows

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_p);
    tma_prefetch_desc(&tmap_q);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], do_cs ? 8 : 4);     // the 4 MMA warps (+ the 4 column-sum warps)
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();      // dependents may begin their prologue ...
  griddep_wait();                   // ... and this kernel touches global memory only after its predecessors are done

  float *dst = p.dwt + ((size_t)split * p.K + k) * p.Cm * p.Cn;
  if (my_chunks > 0) {
    if (warp == 4) {
      // warp-uniform producer loop (see elect_one)
      const int off = k * p.dil - p.pad_l;
      int j = off / p.stride;
      int ph = off - j * p.stride;
      if (ph < 0) { ph += p.stride; j -= 1; }
      int stage = 0;
      uint32_t phase = 0;
      for (int ch = ch_begin; ch < ch_end; ++ch) {
        const int lt = ch % p.n_lt, bg = ch / p.n_lt;
        const int l0 = lt * p.BL, b0 = bg * p.BB;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t *sa = smem + stage * L::STAGE_BYTES;
        uint8_t *sb = sa + 2 * WG_SLAB;
        if (elect_one()) {
          mbar_arrive_expect_tx(&full_bar[stage], (2 + NS) * WG_SLAB);
          tma_load_4d(sa, &tmap_p, &full_bar[stage], m0, 0, l0, b0);
          tma_load_4d(sa + WG_SLAB, &tmap_p, &full_bar[stage], m0 + 64, 0, l0, b0);
#pragma unroll
          for (int s = 0; s < NS; ++s)
            tma_load_4d(sb + s * WG_SLAB, &tmap_q, &full_bar[stage], n0 + 64 * s, ph, l0 + j, b0);
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    } else if (warp < 4) {
      // MMA warpgroup: bf16 x bf16 -> fp32, A and B both MN-major (transposed operands); M half h = P slab h
      const uint32_t smem_base = smem_u32(smem);
      float d[2][BLOCK_N / 2];
      int stage = 0;
      uint32_t phase = 0;
      for (int c = 0; c < my_chunks; ++c) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_base + stage * L::STAGE_BYTES;
        const uint64_t bdesc = make_mnmajor_desc(sa + 2 * WG_SLAB, WG_SLAB);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < WG_ROWS / 16; ++kk) {
          // 16 reduction rows = 2048 bytes -> +128 in the (addr >> 4) field
#pragma unroll
          for (int h = 0; h < 2; ++h)
            Wgmma<BLOCK_N, 1, 1>::mma(d[h], make_mnmajor_desc(sa + h * WG_SLAB, WG_SLAB) + 128 * kk, bdesc + 128 * kk,
                                      (c > 0 || kk > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<BLOCK_N / 2>(d[0]);
        wgmma_fence_regs<BLOCK_N / 2>(d[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      store_wgrad_tile<BLOCK_N>(d, dst, m0, n0, p.Cm, p.Cn);
    } else if (do_cs) {
      // bias gradient: column sums of the P tiles while the tensor core consumes them.  Thread = (8-channel group
      // cg, row residue rg): rows rg, rg+8, ... of both 64-channel slabs, one 16-byte shared load per row.
      const int te = (warp - 5) * 32 + lane;
      const int cg = te & 15, rg = te >> 4;
      const uint32_t col = (uint32_t)(cg >> 3) * WG_SLAB + (uint32_t)(((cg & 7) ^ rg) << 4);
      float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      int stage = 0;
      uint32_t phase = 0;
      for (int c = 0; c < my_chunks; ++c) {
        mbar_wait(&full_bar[stage], phase);
        const uint8_t *sa = smem + stage * L::STAGE_BYTES + col;
#pragma unroll
        for (int i = 0; i < WG_ROWS / 8; ++i) {
          const uint4 q = *reinterpret_cast<const uint4 *>(sa + (rg + 8 * i) * 128);
          const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            cs[2 * j] += __uint_as_float(w[j] << 16);
            cs[2 * j + 1] += __uint_as_float(w[j] & 0xFFFF0000u);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      float *scratch = reinterpret_cast<float *>(smem + L::CS_OFFSET);
#pragma unroll
      for (int j = 0; j < 8; ++j) scratch[rg * 128 + cg * 8 + j] = cs[j];
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float t = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) t += scratch[r * 128 + te];
      p.dbias_part[(size_t)split * p.n_mt * 128 + m0 + te] = t;
    }
  } else if (do_cs && warp >= 5) {
    // empty slice: no rows, zero partial bias gradient
    p.dbias_part[(size_t)split * p.n_mt * 128 + m0 + (warp - 5) * 32 + lane] = 0.f;
  } else if (warp < 4) {
    // empty slice (more splits than row chunks): this CTA still owns its partial tile -> zeros
    const int m = m0 + threadIdx.x;
    if (m < p.Cm) {
      for (int c = 0; c < BLOCK_N; ++c)
        if (n0 + c < p.Cn) dst[(size_t)m * p.Cn + n0 + c] = 0.f;
    }
  }
}

// dwt[K][Cm][Cn] fp32 -> dw[Cm][Cn][K] (transpose=0) or dw[Cn][Cm][K] (transpose=1)
__global__ void __launch_bounds__(256)
tapmajor_to_weight_kernel(const float *__restrict__ dwt, float *__restrict__ dw, int Cm, int Cn, int K,
                          int transpose, int splits) {
  const long total = (long)K * Cm * Cn;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int k = (int)(i % K);
    const long r = i / K;
    int a, c;   // output index (a, c, k): dw[a][c][k]
    a = (int)(r / (transpose ? Cm : Cn));
    c = (int)(r % (transpose ? Cm : Cn));
    const int m = transpose ? c : a, n = transpose ? a : c;
    float acc = 0.f;
    for (int sp = 0; sp < splits; ++sp) acc += dwt[(size_t)sp * total + ((size_t)k * Cm + m) * Cn + n];
    dw[i] = acc;
  }
}

template <int BN>
static int launch_wg(const CUtensorMap &tp, const CUtensorMap &tq, const WgParams &p, cudaStream_t stream) {
  using L = WgSmem<BN>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) {
      set_error("wgrad_tc: cudaFuncSetAttribute(%d bytes): %s", L::TOTAL, cudaGetErrorString(e));
      return 2;
    }
    attr = true;
  }
  const int grid = p.K * p.n_mt * p.n_nt * p.splits;
  launch_pdl(wgrad_tc_kernel<BN>, dim3(grid), dim3(NUM_THREADS), L::TOTAL, stream, tp, tq, p);
  RAVE_CHECK_LAUNCH("wgrad_tc");
  return 0;
}

}  // namespace tc
}  // namespace rave

namespace rave {
namespace tc {
static int wg_block_n(int Cn) {
  // whole 64-channel slabs of the MN-major Q operand; N <= 128: the accumulators live in the MMA warpgroup's registers
  return Cn <= 64 ? 64 : 128;
}
static void wg_geometry(int B, int Cm, int Lp, int Cn, int K, int *BL, int *n_lt, int *n_bg, int *n_mt, int *BN,
                        int *n_nt, int *splits) {
  int bl = WG_ROWS;
  while (bl > Lp && bl > 8) bl >>= 1;
  *BL = bl;
  *n_lt = ceil_div(Lp, bl);
  *n_bg = ceil_div(B, WG_ROWS / bl);
  *n_mt = ceil_div(Cm, 128);
  *BN = wg_block_n(Cn);
  *n_nt = ceil_div(Cn, *BN);
  const int tiles = K * (*n_mt) * (*n_nt);
  const int n_chunks = (*n_lt) * (*n_bg);
  int s = ceil_div(tiles >= 66 ? 132 : 2 * 132, tiles);     // many tiles already: one wave-and-a-bit is enough
  if (s > 32) s = 32;      // every slice writes a full partial tile that the weight-norm backward re-reads
  // ... and a slice of only a few 64-row chunks is all prologue + partial-tile write (the encoder / decoder blocks:
  // 2.4 GFLOP in 40 us): at least 8 chunks per slice
  if (s > n_chunks / 8) s = n_chunks / 8;
  if (s > n_chunks) s = n_chunks;
  if (s < 1) s = 1;
  *splits = s;
}
}  // namespace tc
}  // namespace rave

extern "C" int rave_conv1d_tc_wgrad_splits(int B, int Cm, int Lp, int Cn, int K) {
  int BL, n_lt, n_bg, n_mt, BN, n_nt, splits;
  rave::tc::wg_geometry(B, Cm, Lp, Cn, K, &BL, &n_lt, &n_bg, &n_mt, &BN, &n_nt, &splits);
  return splits;
}

extern "C" int rave_conv1d_tc_wgrad(const void *P, const void *Q, float *dwt, float *dbias, int B, int Cm, int Lp,
                                    int p_pitch, int Cn, int Lq, int q_pitch, int K, int stride, int dil, int pad_l,
                                    void *stream) {
  using namespace rave;
  using namespace rave::tc;
  RAVE_CHECK_ARG(P && Q && dwt, "wgrad_tc: null pointer");
  RAVE_CHECK_ARG(Cm % 8 == 0 && Cn % 8 == 0, "wgrad_tc: channel counts must be multiples of 8 (Cm=%d Cn=%d)", Cm, Cn);
  if (p_pitch <= 0) p_pitch = Lp;
  if (q_pitch <= 0) q_pitch = Lq;
  RAVE_CHECK_ARG(q_pitch >= ceil_div(Lq, stride) * stride,
                 "wgrad_tc: Q pitch %d < Lq %d rounded up to the stride %d (slack rows must be zero)", q_pitch, Lq,
                 stride);
  EncodeTiledFn enc = get_encode_fn();
  RAVE_CHECK_ARG(enc, "wgrad_tc: cuTensorMapEncodeTiled not available");
  cudaStream_t s = (cudaStream_t)stream;

  WgParams p;
  p.B = B; p.Cm = Cm; p.Lp = Lp; p.Cn = Cn; p.Lq = Lq; p.K = K; p.stride = stride; p.dil = dil; p.pad_l = pad_l;
  p.dwt = dwt;
  p.dbias = dbias;
  int BN;
  wg_geometry(B, Cm, Lp, Cn, K, &p.BL, &p.n_lt, &p.n_bg, &p.n_mt, &BN, &p.n_nt, &p.splits);
  p.BB = WG_ROWS / p.BL;

  CUtensorMap tp, tq;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cm, 1, (cuuint64_t)Lp, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2 * p_pitch};
    cuuint32_t box[4] = {64, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(P), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_tc: tensor map P encode failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cn, (cuuint64_t)stride, (cuuint64_t)ceil_div(Lq, stride), (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cn * 2, (cuuint64_t)Cn * 2 * stride, (cuuint64_t)Cn * 2 * q_pitch};
    cuuint32_t box[4] = {64, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tq, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(Q), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_tc: tensor map Q encode failed (%d)", (int)r);
  }
  p.dbias_part = nullptr;
  if (dbias && cudaMallocAsync((void **)&p.dbias_part, sizeof(float) * p.splits * p.n_mt * 128, s) != cudaSuccess) {
    set_error("wgrad_tc: cudaMallocAsync of the bias-gradient partials failed");
    return 2;
  }
  int rc = 1;
  switch (BN) {
    case 64: rc = launch_wg<64>(tp, tq, p, s); break;
    case 128: rc = launch_wg<128>(tp, tq, p, s); break;
    default: set_error("wgrad_tc: no kernel for BLOCK_N=%d", BN);
  }
  if (dbias) {
    if (rc == 0) {
      dbias_sum_kernel<<<ceil_div(Cm, 256), 256, 0, s>>>(p.dbias_part, dbias, p.splits, p.n_mt * 128, Cm);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) {
        set_error("wgrad_tc: dbias_sum launch failed: %s", cudaGetErrorString(e));
        rc = 2;
      } else {
        count_launch();
      }
    }
    cudaFreeAsync(p.dbias_part, s);
  }
  return rc;
}

extern "C" int rave_tapmajor_to_weight_f32(const float *dwt, float *dw, int Cm, int Cn, int K, int transpose,
                                           int splits, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dwt && dw && Cm > 0 && Cn > 0 && K > 0, "tapmajor_to_weight: bad argument");
  const long total = (long)K * Cm * Cn;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  RAVE_CHECK_ARG(splits >= 1, "tapmajor_to_weight: splits must be >= 1");
  tc::tapmajor_to_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dwt, dw, Cm, Cn, K, transpose, splits);
  RAVE_CHECK_LAUNCH("tapmajor_to_weight");
  return 0;
}
#endif  // RAVE_TC_X3_UNIT
