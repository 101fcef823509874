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
// bf16 activated operand of the NEXT conv) reads it row by row while the warpgroup already runs the next tile.  Where
// shared memory allows (plan_smem) there are two such buffers, and the bf16 rows go to a swizzled staging tile that one
// epilogue thread writes out with TMA tensor stores.
// Warp roles: 0-3 = MMA warpgroup, 4 = TMA producer, 5-8 = epilogue.  The input-gradient launches (LeakyReLU' mask,
// bf16 out only) and the forward launches with bias / LeakyReLU and a bf16 output only run the ping-pong kernel instead
// (conv_tc_pp_kernel, conv_tc_pp_fwd_kernel): two MMA warpgroups on alternate tiles, epilogue from registers.  The
// long-k forward launches of that operand set with Cout % 192 == 0 run conv_tc_wide_kernel: two MMA warpgroups on the
// two m64 halves of one 128 x 192 tile.
//
// Replaces: cc.Conv1d.forward = F.pad + F.conv1d -> cuDNN (reference call sites rave/blocks.py:96-108,
// 538-592, 637-692; rave/discriminator.py:99-111), the preceding activation module and the residual add.
#include <string.h>

#include <type_traits>

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
  int act_ld;              // row length (elements) of the bf16 operand tensors the epilogue touches (out_act, res_act):
                           // Cout, or 2*Cout in x3 mode
  int act_cs;              // x3: channels per POSITION of an output row (Cout; Cout/stride when the row holds the phases
                           // of a transposed conv side by side): column n = q*cs + c lives at q*2cs + c (hi), +cs (lo)
  // shared-memory split of this launch (plan_smem): ring stages, accumulator buffers, bf16 output staging tile
  int stages, nacc;
  int stg;                 // 1: out_act rows go through the staging tile and leave by TMA tensor stores
  int acc_off, stg_off, bar_off;
  int ops_off, ops_bytes;  // ping-pong dgrad kernel: the two epilogue operand slots (plan_smem_pp)
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
  // bf16 output staging tile: BLOCK_N / OUT_BOXC boxes of [128 rows][OUT_BOXC channels], each row one swizzle span
  static constexpr int OUT_BOXC = BLOCK_N % 64 == 0 ? 64 : BLOCK_N % 32 == 0 ? 32 : 16;
  static constexpr int OUT_SPAN = OUT_BOXC * 2;
  static constexpr int STG_BYTES = X3 ? 0 : BLOCK_M * BLOCK_N * 2;      // x3 rows ([hi | lo] pairs) keep direct stores
  static constexpr int FIXED = 256 + 1024;                              // barriers + alignment slack
  static constexpr int stages_for(int nacc, int stg) {
    const int s = (SMEM_MAX - FIXED - nacc * ACC_BYTES - stg * STG_BYTES) / STAGE_BYTES;
    return s > 8 ? 8 : s;
  }
};

// Shared-memory split of one launch.  The ring depth the single-buffer layout gives (at most 8) is what the main loop
// needs when a tile has many k-blocks; a tile of kblocks k-blocks cannot use more than kblocks + 1 stages.  The first
// layout that keeps min(that depth, kblocks + 1) stages wins, in this order: two accumulator buffers + the output
// staging tile (the MMA warpgroup hands over a tile without waiting for the epilogue of the previous one; bf16 rows leave
// by TMA), one buffer + staging, one buffer alone (the direct-store epilogue).
template <int BLOCK_N, int BLOCK_K, bool X3>
static void plan_smem(int kblocks, TcParams &p) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  const int base = L::stages_for(1, 0);
  const int need = kblocks + 1 < base ? kblocks + 1 : base;
  p.nacc = 1;
  p.stg = 0;
  if (L::stages_for(2, 1) >= need) { p.nacc = 2; p.stg = 1; }
  else if (L::stages_for(1, 1) >= need) p.stg = 1;
  if (X3) p.stg = 0;
  p.stages = L::stages_for(p.nacc, p.stg);
  p.acc_off = p.stages * L::STAGE_BYTES;
  p.stg_off = p.acc_off + p.nacc * L::ACC_BYTES;
  p.bar_off = p.stg_off + p.stg * L::STG_BYTES;
}

// Byte offset of the 16-byte piece holding channels c .. c + 7 of tile row `row` in the output staging tile: the
// canonical swizzle TMA applies to a box whose rows are one SPAN-byte swizzle span (16-byte piece index XOR address
// bits 7..): the 8 rows one quarter-warp writes land in 8 different bank groups.
template <int BOXC>
__device__ __forceinline__ uint32_t stg_offset(int row, int c) {
  constexpr int SPAN = BOXC * 2;
  const uint32_t line = (uint32_t)row * SPAN;
  const uint32_t piece = (uint32_t)((c % BOXC) >> 3) ^ ((line >> 7) & (SPAN / 16 - 1));
  return (uint32_t)(c / BOXC) * (BLOCK_M * SPAN) + line + (piece << 4);
}

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

// Input-gradient epilogue arithmetic on one column pair (v0, v1), in this order: lrelu_mask, fm_grad, add_bf16_pair.
// Chain rule through the LeakyReLU that produced this conv's operand: the sign bits of the saved bf16 operand pair dm.
__device__ __forceinline__ void lrelu_mask(float &v0, float &v1, uint32_t dm, float slope) {
  if (dm & 0x00008000u) v0 *= slope;
  if (dm & 0x80000000u) v1 *= slope;
}
// Gradient of d0 * sum|h_r - h_f| + d1 * sum|h_r| with respect to h (dm: this row's operand pair, pm: the partner row's).
// LeakyReLU is strictly increasing, so sgn(h_r - h_f) = sgn(a_r - a_f) and sgn(h_r) = sgn(a_r): the saved operands are
// compared as they are.  With t = sgn(a_self - a_partner) both halves get d0 * t (real: d0 sgn(h_r-h_f); fake:
// -d0 sgn(h_r-h_f) = d0 t), real rows d1 sgn(a_self) on top (d1 = 0 on fake rows).  The epilogue is issue-bound on these
// launches: ~6 instructions per element instead of ~20 for the literal form.
__device__ __forceinline__ void fm_grad(float &v0, float &v1, uint32_t dm, uint32_t pm, float d0, float d1) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float as = h ? bf_hi(dm) : bf_lo(dm);
    const float ap = h ? bf_hi(pm) : bf_lo(pm);
    const float t = (as > ap ? 1.f : 0.f) - (as < ap ? 1.f : 0.f);
    const float sr = (as > 0.f ? 1.f : 0.f) - (as < 0.f ? 1.f : 0.f);
    float &v = h ? v1 : v0;
    v = fmaf(d1, sr, fmaf(d0, t, v));
  }
}
// + the bf16 gradient-skip pair rb
__device__ __forceinline__ void add_bf16_pair(float &v0, float &v1, uint32_t rb) {
  v0 += bf_lo(rb);
  v1 += bf_hi(rb);
}

// stg (or null): the output staging tile; out_act then goes there (tile row `row`, channel co - n0) instead of to HBM
template <int CW, bool X3, int BOXC>
__device__ __forceinline__ void tc_epi_chunk(const TcParams &p, uint32_t taddr, int co, bool valid, size_t orow,
                                             int fm_side, uint8_t *stg, int row, int cl) {
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
  acc_ld<CW>(taddr, v);
  if (!valid) return;
  if (p.bias) {
    const float4 *b4 = reinterpret_cast<const float4 *>(p.bias + co);
#pragma unroll
    for (int i = 0; i < CW / 4; ++i) {
      const float4 bb = __ldg(b4 + i);
      v[4 * i] += bb.x; v[4 * i + 1] += bb.y; v[4 * i + 2] += bb.z; v[4 * i + 3] += bb.w;
    }
  }
  if (!X3 && p.dact_src) {
#pragma unroll
    for (int w = 0; w < NW; ++w) lrelu_mask(v[2 * w], v[2 * w + 1], dm[w], p.slope);
  }
  if (!X3 && fm_side) {
    const float d0 = __ldg(p.fm_d), d1 = fm_side > 0 ? __ldg(p.fm_d + 1) : 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) fm_grad(v[2 * w], v[2 * w + 1], dm[w], pm[w], d0, d1);
  }
  if (!X3 && p.res_bf16) {
#pragma unroll
    for (int w = 0; w < NW; ++w) add_bf16_pair(v[2 * w], v[2 * w + 1], rb[w]);
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
    if (!X3 && stg) {
#pragma unroll
      for (int j = 0; j < NW / 4; ++j) sts128(stg + stg_offset<BOXC>(row, cl + 8 * j), pk + 4 * j);
    } else {
      st_words<NW>(p.out_act + offa, pk);
      if (X3) st_words<NW>(p.out_act + offa + cs, pl);
    }
  }
}

template <int BLOCK_N, bool X3, int BOXC>
__device__ __forceinline__ void tc_epilogue(const TcParams &p, uint32_t taddr, int n0, bool valid, size_t orow,
                                            int fm_side, uint8_t *stg, int row) {
  constexpr int MAIN = BLOCK_N / 32 * 32;
  if (X3 && (p.act_cs & 31)) {
    // split-operand rows whose positions are 16 (mod 32) channels wide (capacity-48 transposed convs: 48 channels per
    // position): a 32-column chunk would straddle a [hi | lo] boundary -> 16-column chunks
#pragma unroll 1
    for (int c0 = 0; c0 < BLOCK_N; c0 += 16)
      tc_epi_chunk<16, X3, BOXC>(p, taddr + c0, n0 + c0, valid, orow, fm_side, stg, row, c0);
    return;
  }
#pragma unroll 1
  for (int c0 = 0; c0 < MAIN; c0 += 32)
    tc_epi_chunk<32, X3, BOXC>(p, taddr + c0, n0 + c0, valid, orow, fm_side, stg, row, c0);
  if (MAIN < BLOCK_N) tc_epi_chunk<16, X3, BOXC>(p, taddr + MAIN, n0 + MAIN, valid, orow, fm_side, stg, row, MAIN);
}

// First time step, first batch and first output channel of tile `tile` of the persistent loop (N tiles vary fastest,
// then time tiles, then batch groups)
struct TileCoord {
  int l0, b0, n0;
};
template <int BLOCK_N>
__device__ __forceinline__ TileCoord tile_coord(int tile, const TcParams &p) {
  const int nt = tile % p.n_nt;
  const int mt = tile / p.n_nt;
  const int lt = mt % p.n_lt;
  const int bg = mt / p.n_lt;
  return {lt * p.BL, bg * p.BB, nt * BLOCK_N};
}

// Input row of output row l at tap k: l*stride + k*dil - pad_l = (l + j)*stride + ph, 0 <= ph < stride
struct TapOrigin {
  int j, ph;
};
__device__ __forceinline__ TapOrigin tap_origin(int k, int dil, int pad_l, int stride) {
  const int off = k * dil - pad_l;
  int j = off / stride;
  int ph = off - j * stride;
  if (ph < 0) { ph += stride; j -= 1; }
  return {j, ph};
}

// The operand ring: `stages` slots at the base of shared memory with a full and an empty barrier each; stage / phase =
// the slot of the next k-block and the parity its barriers are at.
struct Ring {
  uint64_t *full, *empty;
  int stages;
  int stage;
  uint32_t phase;
  __device__ __forceinline__ void advance() {
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
};

// Producer (whole warp, elected lane issues): k-block kb of tap k of a tile into the next ring slot once it is free --
// the activation rows from tap origin o, channels kb * BLOCK_K .., and the weight rows of tap k; x3 also the lo halves.
template <int BLOCK_N, int BLOCK_K, bool X3>
__device__ __forceinline__ void produce_kblock(uint8_t *smem, Ring &r, const CUtensorMap *tmap_a,
                                               const CUtensorMap *tmap_b, const TcParams &p, const TileCoord &t,
                                               TapOrigin o, int k, int kb) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  mbar_wait(&r.empty[r.stage], r.phase ^ 1);
  uint8_t *sa = smem + r.stage * L::STAGE_BYTES;
  uint8_t *sb = sa + L::A_BYTES;
  uint64_t *bar = &r.full[r.stage];
  if (elect_one()) {
    mbar_arrive_expect_tx(bar, L::A_BYTES + L::B_BYTES);
    tma_load_4d(sa, tmap_a, bar, kb * BLOCK_K, o.ph, t.l0 + o.j, t.b0);
    tma_load_2d(sb, tmap_b, bar, kb * BLOCK_K, k * p.Cout + t.n0);
    if (X3) {      // lo halves: channels Cin.. of the activation rows, weight slabs K.. (wt is [2][K][Cout][Cin])
      tma_load_4d(sa + L::A_PART, tmap_a, bar, p.Cin + kb * BLOCK_K, o.ph, t.l0 + o.j, t.b0);
      tma_load_2d(sb + L::B_PART, tmap_b, bar, kb * BLOCK_K, (p.K + k) * p.Cout + t.n0);
    }
  }
  __syncwarp();
  r.advance();
}

// The wgmma of k-block kb of a tile from the ring slot at shared address sa, as one committed group: BLOCK_K / 16 steps
// of the two m64 halves (x3: plus lo*hi and hi*lo).  The first step of a tile overwrites the accumulators.  NH = 1: the
// warpgroup issues half h0 alone into d[0] (conv_tc_wide_kernel: the other half is the other warpgroup's).
template <int BLOCK_N, int BLOCK_K, bool X3, int NH = 2>
__device__ __forceinline__ void mma_kblock(float (*d)[BLOCK_N / 2], uint32_t sa, int kb, int h0 = 0) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  constexpr int SWZ = BLOCK_K * 2;
  // rows 64 h .. 64 h + 63 of an operand tile start 64 swizzle spans further: + (64 * SWZ) >> 4 in the address field
  constexpr uint64_t A_HALF = (64 * SWZ) >> 4;
  const uint64_t adesc = make_kmajor_desc(sa, SWZ);
  const uint64_t bdesc = make_kmajor_desc(sa + L::A_BYTES, SWZ);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < BLOCK_K / 16; ++kk) {
    // advance 16 bf16 = 32 bytes inside the swizzle span: +2 in the (addr >> 4) field
#pragma unroll
    for (int h = 0; h < NH; ++h)
      Wgmma<BLOCK_N, 0, 0>::mma(d[h], adesc + (h0 + h) * A_HALF + 2 * kk, bdesc + 2 * kk, (kb > 0 || kk > 0) ? 1u : 0u);
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
}

// Main loop of one tile (MMA warpgroup): its kblocks k-blocks from the ring.  One wgmma group stays in flight: k-block kb
// is issued before the group of kb - 1 is waited for, so the tensor pipe does not drain between k-blocks; a slot is
// released (one arrival per warp) once the group that reads it has completed.  Returns the slot of the last group, which
// is still in flight (mma_drain).  NH, h0: the m64 halves the warpgroup issues (mma_kblock).
template <int BLOCK_N, int BLOCK_K, bool X3, int NH = 2>
__device__ __forceinline__ int mma_mainloop(float (*d)[BLOCK_N / 2], uint32_t smem_base, Ring &r, int kblocks,
                                            int lane, int h0 = 0) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  int prev = 0;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(&r.full[r.stage], r.phase);
    mma_kblock<BLOCK_N, BLOCK_K, X3, NH>(d, smem_base + r.stage * L::STAGE_BYTES, kb, h0);
    wgmma_wait<1>();                                         // the group of k-block kb - 1 has completed
    if (kb > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&r.empty[prev]);            // this warp's MMAs no longer read that slot
    }
    prev = r.stage;
    r.advance();
  }
  return prev;
}

// End of a tile's main loop: wait for its last wgmma group, then release that group's slot
template <int BLOCK_N, int NH = 2>
__device__ __forceinline__ void mma_drain(float (*d)[BLOCK_N / 2], const Ring &r, int prev, int lane) {
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < NH; ++h) wgmma_fence_regs<BLOCK_N / 2>(d[h]);
  __syncwarp();
  if (lane == 0) mbar_arrive(&r.empty[prev]);
}

template <int BLOCK_N, int BLOCK_K, bool X3>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_o, const TcParams p) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, X3>;
  const int STAGES = p.stages;
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N >= 16 && BLOCK_N <= 128, "invalid wgmma N");

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + p.bar_off);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *tfull_bar = empty_bar + STAGES;      // MMA warpgroup -> epilogue: accumulator buffer b holds a tile
  uint64_t *tempty_bar = tfull_bar + 2;          // epilogue -> MMA warpgroup: buffer b has been read
  uint8_t *stg = (!X3 && p.stg) ? smem + p.stg_off : nullptr;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg * p.n_nt;
  const int kblocks = p.K * p.num_kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (stg) tma_prefetch_desc(&tmap_o);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);               // one arrival per MMA warp
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&tfull_bar[b], 128);
      mbar_init(&tempty_bar[b], 4);
    }
    fence_barrier_init();
    acc_bind(smem + p.acc_off, L::ACC_LD);       // nacc buffers back to back: buffer b = rows 128 b ..
  }
  __syncthreads();
  griddep_launch_dependents();      // dependents may begin their prologue ...
  griddep_wait();                   // ... and this kernel touches global memory only after its predecessors are done

  Ring ring{full_bar, empty_bar, STAGES, 0, 0};
  if (warp == 4) {
    // =========================== TMA producer (warp-uniform loop, elected lane issues) ===========================
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      for (int k = 0; k < p.K; ++k) {
        const TapOrigin o = tap_origin(k, p.dil, p.pad_l, p.stride);
        for (int kb = 0; kb < p.num_kb; ++kb)
          produce_kblock<BLOCK_N, BLOCK_K, X3>(smem, ring, &tmap_a, &tmap_b, p, t, o, k, kb);
      }
    }
  } else if (warp < 4) {
    // =========================== MMA warpgroup ===========================
    const uint32_t smem_base = smem_u32(smem);
    float d[2][BLOCK_N / 2];
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int prev = mma_mainloop<BLOCK_N, BLOCK_K, X3>(d, smem_base, ring, kblocks, lane);
      mma_drain<BLOCK_N>(d, ring, prev, lane);
      const int buf = p.nacc == 2 ? (it & 1) : 0;
      const uint32_t use = p.nacc == 2 ? (it >> 1) : it;         // earlier tiles handed over through this buffer
      mbar_wait(&tempty_bar[buf], (use & 1) ^ 1);                // the epilogue has read the buffer's previous tile
      acc_store<BLOCK_N>(d, threadIdx.x, 0, 128 * buf);
      mbar_arrive(&tfull_bar[buf]);
    }
  } else {
    // =========================== epilogue (4 warps) ===========================
    constexpr int BOXC = L::OUT_BOXC;
    const int quad = warp & 3;           // rows quad * 32 .. quad * 32 + 31 of the tile
    const int row = quad * 32 + lane;    // row of the 128-row tile
    const bool issuer = threadIdx.x == 160;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      const int n0 = t.n0;
      const int b = t.b0 + row / p.BL;
      const int l = t.l0 + row % p.BL;
      const bool valid = (b < p.B) && (l < p.Lout);
      const size_t orow = (size_t)b * p.out_rows + (size_t)l * p.out_row_stride + p.out_row_offset;

      const int buf = p.nacc == 2 ? (it & 1) : 0;
      const uint32_t use = p.nacc == 2 ? (it >> 1) : it;
      if (stg) {                         // the previous tile's tensor stores have read the staging tile
        if (issuer) bulk_wait_read<0>();
        named_bar_sync(1, 128);
      }
      mbar_wait(&tfull_bar[buf], use & 1);
      const uint32_t taddr = (uint32_t)(128 * buf + quad * 32) << 16;
      tc_epilogue<BLOCK_N, X3, BOXC>(p, taddr, n0, valid, orow, p.fm_d ? (b < p.fm_bh ? 1 : -1) : 0, stg, row);
      __syncwarp();
      if (lane == 0) mbar_arrive(&tempty_bar[buf]);
      if (stg) {
        // rows past Lout and batches past B fall outside the tensor map and are not written
        fence_proxy_async();             // generic-proxy shared-memory writes -> TMA
        named_bar_sync(1, 128);
        if (issuer) {
#pragma unroll
          for (int c = 0; c < BLOCK_N; c += BOXC)
            tma_store_3d(&tmap_o, stg + (c / BOXC) * (BLOCK_M * L::OUT_SPAN), n0 + c, t.l0, t.b0);
          bulk_commit();
        }
      }
    }
    if (stg && issuer) bulk_wait_all();
  }
}

// =============================================================================================
// Ping-pong kernel.  The launches whose epilogue applies the LeakyReLU' mask (dact_src), optionally with the fused
// feature-matching term and the bf16 gradient skip, and writes bf16 only (the input gradients of every chain) read up
// to three operand tiles per output tile; in conv_tc_kernel that epilogue is as long as the main loop and the MMAs wait
// for it.  Here two MMA warpgroups take alternate tiles of the persistent loop: each runs a whole 128 x BLOCK_N tile
// (the same wgmma sequence as conv_tc_kernel) and then its epilogue straight from its accumulator registers while the
// other one runs its main loop; an ordering barrier pair hands the tensor pipe from one warpgroup to the other.  When
// the producer starts a tile it also loads the tile's epilogue operands with TMA into that warpgroup's operand slot,
// on a barrier of their own, so they land during the main loop; the bf16 result replaces the mask in the slot (same
// swizzled position) and leaves by TMA tensor stores.
// The forward launches with bias / LeakyReLU and a bf16 output only (the discriminator convs) run the same kernel
// with the forward epilogue: no operands to load, the slot holds the output tile alone.  On the short-k launches
// conv_tc_kernel's four epilogue warps (one per SM sub-partition, fed through a 64 KB fp32 hand-over buffer) bound
// the launch; here eight warps run the epilogue from registers.
// Warp roles: warpgroup 0 = TMA producer (warp 0; warps 1-3 leave after giving their registers back), warpgroups 1
// and 2 = MMA + epilogue.
// =============================================================================================
constexpr int PP_THREADS = 384;

// Operand set of a ping-pong instance (template argument of conv_tc_pp_body).  Input gradient: LeakyReLU' mask,
// + feature-matching partner rows (PP_FM), + gradient skip (PP_RS).  Forward (PP_FWD): + bias (PP_BIAS), LeakyReLU
// (PP_LEAKY).
enum PpEpi : int { PP_FM = 1, PP_RS = 2, PP_FWD = 4, PP_BIAS = 8, PP_LEAKY = 16 };

// Epilogue of one tile from the accumulator registers of warpgroup thread (w, lane).  slot = [mask | partner (FM) |
// gradient skip (RS)] tiles, each BLOCK_N / BOXC boxes of [128 rows][BOXC channels] in the canonical swizzle.  Per
// element the same fp32 sequence as tc_epi_chunk (lrelu_mask, fm_grad, add_bf16_pair), one rounding to bf16.
template <int BLOCK_N, int BOXC, bool FM, bool RS>
__device__ __forceinline__ void pp_epilogue(float (*d)[BLOCK_N / 2], uint8_t *slot, const TcParams &p, int w, int lane,
                                            int b0) {
  constexpr int TILE_BYTES = BLOCK_M * BLOCK_N * 2;
  uint8_t *part = slot + TILE_BYTES;
  uint8_t *skip = slot + (FM ? 2 : 1) * TILE_BYTES;
  constexpr int SPAN = BOXC * 2, JB = BOXC / 8;          // 16-byte pieces per box row
  const float d0 = FM ? __ldg(p.fm_d) : 0.f, d1 = FM ? __ldg(p.fm_d + 1) : 0.f;
  // wgmma fragment: d[h][4 j + 2 r + {0, 1}] = row 64 h + 16 w + lane / 4 + 8 r, columns 8 j + 2 (lane % 4) + {0, 1}.
  // The four rows of a thread are 8 apart, so they share the swizzle (piece index XOR row bits that a multiple of 8
  // rows does not change): the word of column 8 j + 2 (lane % 4) sits at base ^ (j % JB) << 4, plus a whole box per
  // JB pieces and a constant per row -- JB registers of addresses instead of one per element.
  const uint32_t base = stg_offset<BOXC>(16 * w + (lane >> 2), 0) + 4 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = 64 * h + 16 * w + (lane >> 2) + 8 * r;
      const float d1r = (FM && b0 + row / p.BL < p.fm_bh) ? d1 : 0.f;     // d1 sgn(a_r) on real rows only
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const uint32_t off = (base ^ (uint32_t)((j % JB) << 4)) + (j / JB) * (BLOCK_M * SPAN) + (64 * h + 8 * r) * SPAN;
        float v0 = d[h][4 * j + 2 * r], v1 = d[h][4 * j + 2 * r + 1];
        const uint32_t dm = *reinterpret_cast<const uint32_t *>(slot + off);
        lrelu_mask(v0, v1, dm, p.slope);
        if (FM) fm_grad(v0, v1, dm, *reinterpret_cast<const uint32_t *>(part + off), d0, d1r);
        if (RS) add_bf16_pair(v0, v1, *reinterpret_cast<const uint32_t *>(skip + off));
        __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        *reinterpret_cast<uint32_t *>(slot + off) = *reinterpret_cast<uint32_t *>(&o);
      }
    }
  }
}

// Forward epilogue of one tile from the accumulator registers into the output slot (the boxes and fragment mapping of
// pp_epilogue).  Per element the fp32 sequence of tc_epi_chunk: + bias[co], max(v, slope v) for LeakyReLU, one rounding
// to bf16.  Column pair j outermost: one bias load per pair serves the thread's four rows.  NH, h0: the m64 halves the
// warpgroup holds (mma_kblock); with NH = 1 a thread has two rows.
template <int BLOCK_N, int BOXC, bool BIAS, bool LEAKY, int NH = 2>
__device__ __forceinline__ void pp_fwd_epilogue(float (*d)[BLOCK_N / 2], uint8_t *slot, const TcParams &p, int w,
                                                int lane, int n0, int h0 = 0) {
  constexpr int SPAN = BOXC * 2, JB = BOXC / 8;
  const uint32_t base = stg_offset<BOXC>(16 * w + (lane >> 2), 0) + 4 * (lane & 3);
  const uint32_t sslot = smem_u32(slot);
  const float2 *bias = reinterpret_cast<const float2 *>(p.bias + n0 + 2 * (lane & 3));   // columns 8 j + 2 (lane % 4)
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const float2 bb = BIAS ? __ldg(bias + 4 * j) : make_float2(0.f, 0.f);
    const uint32_t col = (base ^ (uint32_t)((j % JB) << 4)) + (j / JB) * (BLOCK_M * SPAN);
#pragma unroll
    for (int h = 0; h < NH; ++h) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float v0 = d[h][4 * j + 2 * r], v1 = d[h][4 * j + 2 * r + 1];
        if (BIAS) {
          v0 += bb.x;
          v1 += bb.y;
        }
        if (LEAKY) {
          v0 = fmaxf(v0, v0 * p.slope);
          v1 = fmaxf(v1, v1 * p.slope);
        }
        __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        // volatile: each store stays next to its arithmetic (with plain stores ptxas ran all of a tile's arithmetic
        // ahead of the stores and spilled tile-loop invariants at BLOCK_N = 128)
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sslot + col + (64 * (h0 + h) + 8 * r) * SPAN),
                     "r"(*reinterpret_cast<uint32_t *>(&o))
                     : "memory");
      }
    }
  }
}

// The ping-pong kernel of operand set E (PpEpi flags).  Tensor maps: a, b = MMA operands, o = bf16 output rows;
// input gradients also m = mask, pm = partner rows (PP_FM), r = gradient skip (PP_RS).
template <int BLOCK_N, int BLOCK_K, int E>
__device__ __forceinline__ void conv_tc_pp_body(const CUtensorMap *tmap_a, const CUtensorMap *tmap_b,
                                                const CUtensorMap *tmap_m, const CUtensorMap *tmap_p,
                                                const CUtensorMap *tmap_r, const CUtensorMap *tmap_o,
                                                const TcParams &p) {
  using L = SmemLayout<BLOCK_N, BLOCK_K, false>;
  constexpr int BOXC = L::OUT_BOXC;
  constexpr int BOX_BYTES = BLOCK_M * L::OUT_SPAN;          // one [128 rows][BOXC channels] box
  constexpr int TILE_BYTES = BLOCK_M * BLOCK_N * 2;         // one operand tile
  constexpr bool FWD = E & PP_FWD, FM = E & PP_FM, RS = E & PP_RS;
  const int STAGES = p.stages;
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N >= 16 && BLOCK_N <= 128, "invalid wgmma N");
  static_assert(!FWD || !(FM || RS), "the forward epilogue has no gradient operands");

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + p.bar_off);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *ofull_bar = empty_bar + STAGES;      // producer -> warpgroup c: its operand slot holds the tile's operands
  uint64_t *oempty_bar = ofull_bar + 2;          // warpgroup c -> producer (forward: -> itself): the tensor stores
                                                 // have read the slot
  uint64_t *order_bar = oempty_bar + 2;          // warpgroup 1 - c -> c: c may issue its main loop

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg * p.n_nt;
  const int kblocks = p.K * p.num_kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmap_a);
    tma_prefetch_desc(tmap_b);
    tma_prefetch_desc(tmap_o);
    if constexpr (!FWD) tma_prefetch_desc(tmap_m);
    if constexpr (FM) tma_prefetch_desc(tmap_p);
    if constexpr (RS) tma_prefetch_desc(tmap_r);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);               // one arrival per MMA warp of the consuming warpgroup
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(&ofull_bar[c], 1);
      mbar_init(&oempty_bar[c], 1);
      mbar_init(&order_bar[c], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();
  griddep_wait();

  if (wg == 0) {
    // =========================== TMA producer (warp-uniform loop, elected lane issues) ===========================
    warpgroup_reg_dealloc<56>();
    if (warp != 0) return;
    Ring ring{full_bar, empty_bar, STAGES, 0, 0};
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      const int c = it & 1;                        // consumer warpgroup of this tile
      for (int k = 0; k < p.K; ++k) {
        const TapOrigin o = tap_origin(k, p.dil, p.pad_l, p.stride);
        for (int kb = 0; kb < p.num_kb; ++kb) {
          produce_kblock<BLOCK_N, BLOCK_K, false>(smem, ring, tmap_a, tmap_b, p, t, o, k, kb);
          if (!FWD && k == 0 && kb == 0) {
            // The tile's epilogue operands, behind its first k-block, into warpgroup c's slot once the tensor stores of
            // that warpgroup's previous tile have read it.  A box past Lout / B is zero-filled and still counts in full.
            mbar_wait(&oempty_bar[c], ((it >> 1) & 1) ^ 1);
            uint8_t *slot = smem + p.ops_off + c * p.ops_bytes;
            if (elect_one()) {
              mbar_arrive_expect_tx(&ofull_bar[c], p.ops_bytes);
              for (int cb = 0; cb < BLOCK_N / BOXC; ++cb) {
                tma_load_3d(slot + cb * BOX_BYTES, tmap_m, &ofull_bar[c], t.n0 + cb * BOXC, t.l0, t.b0);
                if (FM) {
                  // partner rows one batch at a time: a batch group may straddle the [real; fake] boundary
                  for (int i = 0; i < p.BB; ++i) {
                    const int b = t.b0 + i;
                    const int pb = p.fm_bh > 0 ? (b < p.fm_bh ? b + p.fm_bh : b - p.fm_bh) : b;
                    tma_load_3d(slot + TILE_BYTES + cb * BOX_BYTES + i * p.BL * L::OUT_SPAN, tmap_p, &ofull_bar[c],
                                t.n0 + cb * BOXC, t.l0, pb);
                  }
                }
                if (RS)
                  tma_load_3d(slot + (FM ? 2 : 1) * TILE_BYTES + cb * BOX_BYTES, tmap_r, &ofull_bar[c],
                              t.n0 + cb * BOXC, t.l0, t.b0);
              }
            }
            __syncwarp();
          }
        }
      }
    }
  } else {
    // =========================== MMA + epilogue warpgroups 1, 2 ===========================
    warpgroup_reg_alloc<224>();
    const int c = wg - 1;
    const int w = warp & 3;
    const bool issuer = (threadIdx.x & 127) == 0;
    const uint32_t smem_base = smem_u32(smem);
    uint8_t *slot = smem + p.ops_off + c * p.ops_bytes;
    float d[2][BLOCK_N / 2];
    int u = 0;                                     // tiles this warpgroup has run
    for (int tile = blockIdx.x + c * gridDim.x; tile < num_tiles; tile += 2 * gridDim.x, ++u) {
      const int it = 2 * u + c;                    // position of the tile in the CTA's sequence
      const uint32_t g0 = (uint32_t)it * (uint32_t)kblocks;      // ring position of its first k-block
      Ring ring{full_bar, empty_bar, STAGES, (int)(g0 % (uint32_t)STAGES), (g0 / (uint32_t)STAGES) & 1};
      if (it > 0) mbar_wait(&order_bar[c], ((it - 1) >> 1) & 1);  // the other warpgroup has issued tile it - 1
      const int prev = mma_mainloop<BLOCK_N, BLOCK_K, false>(d, smem_base, ring, kblocks, lane);
      __syncwarp();
      if (lane == 0) mbar_arrive(&order_bar[c ^ 1]);             // every MMA of this tile is issued
      mma_drain<BLOCK_N>(d, ring, prev, lane);

      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      if constexpr (FWD) {
        mbar_wait(&oempty_bar[c], (u & 1) ^ 1);    // the tensor stores of this warpgroup's previous tile read the slot
        pp_fwd_epilogue<BLOCK_N, BOXC, (E & PP_BIAS) != 0, (E & PP_LEAKY) != 0>(d, slot, p, w, lane, t.n0);
      } else {
        mbar_wait(&ofull_bar[c], u & 1);
        pp_epilogue<BLOCK_N, BOXC, FM, RS>(d, slot, p, w, lane, t.b0);
      }
      // rows past Lout and batches past B fall outside the tensor map and are not written
      fence_proxy_async();
      named_bar_sync(1 + c, 128);
      if (issuer) {
#pragma unroll
        for (int cb = 0; cb < BLOCK_N / BOXC; ++cb)
          tma_store_3d(tmap_o, slot + cb * BOX_BYTES, t.n0 + cb * BOXC, t.l0, t.b0);
        bulk_commit();
        bulk_wait_read<0>();
        mbar_arrive(&oempty_bar[c]);
      }
    }
    if (issuer) bulk_wait_all();
  }
}

// Input gradients.  FM, RS: fm_d, res_bf16 set.  One instance per operand set: the epilogue compiled once for run-time
// flags made the v2 step slower (DESIGN section 5.3).
template <int BLOCK_N, int BLOCK_K, bool FM, bool RS>
__global__ void __launch_bounds__(PP_THREADS, 1)
conv_tc_pp_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_m, const __grid_constant__ CUtensorMap tmap_p,
                  const __grid_constant__ CUtensorMap tmap_r, const __grid_constant__ CUtensorMap tmap_o,
                  const TcParams p) {
  conv_tc_pp_body<BLOCK_N, BLOCK_K, (FM ? PP_FM : 0) | (RS ? PP_RS : 0)>(&tmap_a, &tmap_b, &tmap_m, &tmap_p, &tmap_r,
                                                                         &tmap_o, p);
}

// Forward.  BIAS: bias set, LEAKY: act = RAVE_ACT_LEAKY; one instance per operand set as above.
template <int BLOCK_N, int BLOCK_K, bool BIAS, bool LEAKY>
__global__ void __launch_bounds__(PP_THREADS, 1)
conv_tc_pp_fwd_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_o, const TcParams p) {
  conv_tc_pp_body<BLOCK_N, BLOCK_K, PP_FWD | (BIAS ? PP_BIAS : 0) | (LEAKY ? PP_LEAKY : 0)>(
      &tmap_a, &tmap_b, nullptr, nullptr, nullptr, &tmap_o, p);
}

// =============================================================================================
// Wide forward kernel.  The long-k forward launches of the PP_FWD operand set whose Cout is a multiple of 192 (the
// discriminators' layers 2-4) run 128 x 192 tiles: warpgroups 1 and 2 both work on every tile, warpgroup 1 on rows
// 0-63 and warpgroup 2 on rows 64-127, each issuing m64n192k16 from the same ring stage.  An activation tile is then
// loaded once per 192 output channels instead of once per 96 or 128, and each stage's weight tile feeds two m64 blocks
// per k16 step as in conv_tc_kernel, so shared memory serves fewer operand bytes per MMA.  Each output element gets
// conv_tc_kernel's k16 steps in the same order; the epilogue is pp_fwd_epilogue's, so the bf16 output is the same.
// Warp roles as in conv_tc_pp_body: warpgroup 0 = TMA producer (warp 0), warpgroups 1 and 2 = MMA + epilogue.  The ring
// (produce_kblock, mma_mainloop) is shared: a stage is free once all 8 MMA warps have released it.  Both warpgroups
// write their rows into one bf16 output slot (128 x 192, 48 KB); after a named barrier one thread stores it by TMA.
// Before the next tile's epilogue that thread waits until the stores have read the slot and arms oempty, which both
// warpgroups wait on before they write the slot again.  The epilogue does not overlap the MMAs of the CTA, so the
// kernel only takes launches with many k-blocks per tile (wide_stages).
// =============================================================================================
constexpr int WIDE_N = 192;

template <int BLOCK_K, bool BIAS, bool LEAKY>
__global__ void __launch_bounds__(PP_THREADS, 1)
conv_tc_wide_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const __grid_constant__ CUtensorMap tmap_o, const TcParams p) {
  constexpr int BLOCK_N = WIDE_N;
  using L = SmemLayout<BLOCK_N, BLOCK_K, false>;
  constexpr int BOXC = L::OUT_BOXC;
  constexpr int BOX_BYTES = BLOCK_M * L::OUT_SPAN;
  const int STAGES = p.stages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + p.bar_off);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *oempty_bar = empty_bar + STAGES;     // store issuer -> both warpgroups: the tensor stores have read the slot

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.n_lt * p.n_bg * p.n_nt;
  const int kblocks = p.K * p.num_kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_o);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);               // one arrival per MMA warp of both warpgroups
    }
    mbar_init(oempty_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();
  griddep_wait();

  Ring ring{full_bar, empty_bar, STAGES, 0, 0};
  if (wg == 0) {
    // =========================== TMA producer (warp-uniform loop, elected lane issues) ===========================
    warpgroup_reg_dealloc<56>();
    if (warp != 0) return;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      for (int k = 0; k < p.K; ++k) {
        const TapOrigin o = tap_origin(k, p.dil, p.pad_l, p.stride);
        for (int kb = 0; kb < p.num_kb; ++kb)
          produce_kblock<BLOCK_N, BLOCK_K, false>(smem, ring, &tmap_a, &tmap_b, p, t, o, k, kb);
      }
    }
  } else {
    // =========================== MMA + epilogue warpgroups 1, 2: rows 64 h .. 64 h + 63 ===========================
    warpgroup_reg_alloc<224>();
    const int h = wg - 1;
    const int w = warp & 3;
    const bool issuer = threadIdx.x == 128;
    const uint32_t smem_base = smem_u32(smem);
    uint8_t *slot = smem + p.ops_off;
    float d[1][BLOCK_N / 2];
    int u = 0;                                     // tiles this CTA has run
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++u) {
      const int prev = mma_mainloop<BLOCK_N, BLOCK_K, false, 1>(d, smem_base, ring, kblocks, lane, h);
      mma_drain<BLOCK_N, 1>(d, ring, prev, lane);
      const TileCoord t = tile_coord<BLOCK_N>(tile, p);
      // the tensor stores of the previous tile have read the slot (they ran during this tile's main loop)
      if (issuer && u > 0) {
        bulk_wait_read<0>();
        mbar_arrive(oempty_bar);
      }
      mbar_wait(oempty_bar, (u & 1) ^ 1);
      pp_fwd_epilogue<BLOCK_N, BOXC, BIAS, LEAKY, 1>(d, slot, p, w, lane, t.n0, h);
      // rows past Lout and batches past B fall outside the tensor map and are not written
      fence_proxy_async();
      named_bar_sync(1, 256);
      if (issuer) {
#pragma unroll
        for (int cb = 0; cb < BLOCK_N / BOXC; ++cb)
          tma_store_3d(&tmap_o, slot + cb * BOX_BYTES, t.n0 + cb * BOXC, t.l0, t.b0);
        bulk_commit();
      }
    }
    if (issuer) bulk_wait_all();
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
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

// Tile geometry of a launch: M tiles of BB batches x BL time steps, BN (BLOCK_N) output channels per N tile, num_kb
// k-blocks of BK (BLOCK_K) input channels per tap.  BK = 0 or BN = 0: no kernel covers the shape.
struct TcGeometry {
  int BK, BL, BB, n_lt, n_bg, BN, n_nt, num_kb;
};
static TcGeometry tc_geometry(int B, int Cin, int Cout, int Lout) {
  TcGeometry g;
  g.BK = pick_block_k(Cin);
  g.BL = 128;
  while (g.BL > Lout && g.BL > 8) g.BL >>= 1;   // power of two <= max(Lout, 8)
  g.BB = 128 / g.BL;
  g.n_lt = ceil_div(Lout, g.BL);
  g.n_bg = ceil_div(B, g.BB);
  g.BN = pick_block_n(Cout, (long)g.n_lt * g.n_bg);
  g.n_nt = g.BN ? Cout / g.BN : 0;
  g.num_kb = g.BK ? ceil_div(Cin, g.BK) : 0;
  return g;
}

// f(BK, BN) with std::integral_constant arguments, for each (BLOCK_K, BLOCK_N) pair the kernels are built for; any other
// pair is an error (1)
template <int BK, typename F>
static int visit_block_n(int BN, F &f) {
  using std::integral_constant;
  switch (BN) {
    case 128: return f(integral_constant<int, BK>(), integral_constant<int, 128>());
    case 96: return f(integral_constant<int, BK>(), integral_constant<int, 96>());
    case 64: return f(integral_constant<int, BK>(), integral_constant<int, 64>());
    case 48: return f(integral_constant<int, BK>(), integral_constant<int, 48>());
    case 32: return f(integral_constant<int, BK>(), integral_constant<int, 32>());
    case 16: return f(integral_constant<int, BK>(), integral_constant<int, 16>());
  }
  set_error("conv1d_tc: no kernel for BLOCK_N=%d", BN);
  return 1;
}
template <typename F>
static int visit_tile(int BK, int BN, F &&f) {
  switch (BK) {
    case 64: return visit_block_n<64>(BN, f);
    case 32: return visit_block_n<32>(BN, f);
    case 16: return visit_block_n<16>(BN, f);
  }
  set_error("conv1d_tc: no kernel for BLOCK_K=%d", BK);
  return 1;
}

// bf16 rows (c, l, b) over [B][out_rows][Cout] from row out_row_offset on: row l of batch b is
// b * out_rows + l * out_row_stride + out_row_offset; the extents Lout and B clip the rows of a ragged tile.  Boxes of
// [box_b batches][BL rows][OUT_BOXC channels], each row one swizzle span.
template <int BN>
static int encode_rows_map(CUtensorMap *m, const __nv_bfloat16 *base, const TcParams &p, int box_b) {
  using L = SmemLayout<BN, 64, false>;
  const cuuint64_t dims[3] = {(cuuint64_t)p.Cout, (cuuint64_t)p.Lout, (cuuint64_t)p.B};
  const cuuint64_t strides[2] = {(cuuint64_t)p.Cout * 2 * p.out_row_stride, (cuuint64_t)p.Cout * 2 * p.out_rows};
  const cuuint32_t box[3] = {(cuuint32_t)L::OUT_BOXC, (cuuint32_t)p.BL, (cuuint32_t)box_b};
  const CUresult r = encode_bf16_map(m, 3, base + (size_t)p.out_row_offset * p.Cout, dims, strides, box,
                                     swizzle_enum(L::OUT_SPAN), CU_TENSOR_MAP_L2_PROMOTION_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("conv1d_tc: bf16 row tensor map encode failed (%d)", (int)r);
    return 1;
  }
  return 0;
}

// BLOCK_N = 96 at BLOCK_K = 64: ptxas spills tile-loop invariants of every input-gradient ping-pong instance, so none
// is built and conv_tc_kernel runs these launches
template <int BN, int BK, bool FWD>
constexpr bool pp_built = FWD || !(BN == 96 && BK == 64);

// Ring stages of a ping-pong launch whose operand slots hold nops tiles each (mask, + partner rows with fm_d, + gradient
// skip with res_bf16, or the forward output alone: [128][BLOCK_N] bf16 each); the ring gets the rest (at most 8
// stages).  0: the launch runs conv_tc_kernel -- no instance for the tile, or fewer than 2 stages fit (mask + partner +
// skip at BLOCK_N = 128, BLOCK_K = 64).
template <int BN, int BK, bool FWD>
constexpr int pp_stages(int nops) {
  using L = SmemLayout<BN, BK, false>;
  if (!pp_built<BN, BK, FWD>) return 0;
  const int s = (SMEM_MAX - L::FIXED - 2 * nops * BLOCK_M * BN * 2) / L::STAGE_BYTES;
  return s < 2 ? 0 : s > 8 ? 8 : s;
}

// Ring stages of a forward launch (bias / LeakyReLU -> bf16 only) of kblocks k-blocks per tile on the ping-pong
// kernel; 0: it runs conv_tc_kernel.  The ping-pong kernel takes the launch when its ring is at least as deep as the
// one plan_smem gives conv_tc_kernel and either the tile has at most 24 k-blocks or BLOCK_N = 128 (there the 64 KB
// hand-over buffer leaves conv_tc_kernel 3-4 stages; the ping-pong slot leaves 5).  Tensor-bound launches of 36-72
// k-blocks per tile at BLOCK_N = 64 and 96 measured 8-22 % slower on the ping-pong kernel (conv_tc_kernel already hides
// their epilogue behind the main loop and keeps 7-8 stages); see DESIGN section 5.6.
template <int BN, int BK>
static int pp_fwd_stages(int kblocks) {
  const int s = pp_stages<BN, BK, true>(1);
  TcParams q;
  plan_smem<BN, BK, false>(kblocks, q);
  return s >= q.stages && (BN == 128 || kblocks <= 24) ? s : 0;
}

// Wide forward kernel (conv_tc_wide_kernel): BLOCK_K of a launch of Cin input channels, and its ring stages next to the
// 48 KB output slot (4 at BLOCK_K = 64, 8 at BLOCK_K = 32).
static int wide_block_k(int Cin) { return pick_block_k(Cin); }
template <int BK>
constexpr int wide_ring_stages() {
  using L = SmemLayout<WIDE_N, BK, false>;
  const int s = (SMEM_MAX - L::FIXED - L::STG_BYTES) / L::STAGE_BYTES;
  return s > 8 ? 8 : s;
}
// Fewest k-blocks per tile for which a forward launch (bias / LeakyReLU -> bf16 only) with Cout % 192 == 0 runs the wide
// kernel: its epilogue does not overlap the CTA's MMAs, so the short-k launches stay on the ping-pong kernel.  Measured
// (DESIGN section 5.6): every v2 launch of 15-90 k-blocks per tile took 5-30 % less time than on the ping-pong kernel or
// conv_tc_kernel; one of 12 k-blocks broke even.
constexpr int WIDE_MIN_KBLOCKS = 12;
// Instances: BLOCK_K = 64 and 32 (Cin a multiple of 32).
static int wide_stages(int Cin, int Cout, int K) {
  const int BK = wide_block_k(Cin);
  if (BK < 32 || Cout % WIDE_N || K * ceil_div(Cin, BK) < WIDE_MIN_KBLOCKS) return 0;
  return BK == 64 ? wide_ring_stages<64>() : wide_ring_stages<32>();
}

template <int BK>
static int launch_wide(const CUtensorMap &ta, const CUtensorMap &tb, TcParams p, int stages, cudaStream_t stream) {
  using L = SmemLayout<WIDE_N, BK, false>;
  p.stages = stages;
  p.ops_bytes = L::STG_BYTES;
  p.ops_off = p.stages * L::STAGE_BYTES;
  p.bar_off = p.ops_off + p.ops_bytes;
  const int grid = persistent_grid(p.n_lt * p.n_bg * p.n_nt), smem = p.bar_off + L::FIXED;
  CUtensorMap to;
  if (encode_rows_map<WIDE_N>(&to, p.out_act, p, p.BB)) return 1;
  const auto go = [&](auto bias, auto leaky) {
    return launch_tc<conv_tc_wide_kernel<BK, decltype(bias)::value, decltype(leaky)::value>>(
        "conv1d_tc", grid, PP_THREADS, smem, stream, ta, tb, to, p);
  };
  const std::true_type y;
  const std::false_type n;
  const bool leaky = p.act == RAVE_ACT_LEAKY;
  return p.bias ? (leaky ? go(y, y) : go(y, n)) : (leaky ? go(n, y) : go(n, n));
}

// FWD: a forward launch (bias / LeakyReLU; the slot holds the output tile alone), else an input-gradient launch
template <int BN, int BK, bool FWD>
static int launch_pp(const CUtensorMap &ta, const CUtensorMap &tb, TcParams p, int stages, cudaStream_t stream) {
  using L = SmemLayout<BN, BK, false>;
  p.stages = stages;
  p.ops_bytes = (1 + (p.fm_d ? 1 : 0) + (p.res_bf16 ? 1 : 0)) * BLOCK_M * BN * 2;
  p.ops_off = p.stages * L::STAGE_BYTES;
  p.bar_off = p.ops_off + 2 * p.ops_bytes;
  const int grid = persistent_grid(p.n_lt * p.n_bg * p.n_nt), smem = p.bar_off + L::FIXED;
  const std::true_type y;
  const std::false_type n;
  CUtensorMap tm, tp, tr, to;
  if (encode_rows_map<BN>(&to, p.out_act, p, p.BB)) return 1;
  if constexpr (FWD) {
    const auto go = [&](auto bias, auto leaky) {
      return launch_tc<conv_tc_pp_fwd_kernel<BN, BK, decltype(bias)::value, decltype(leaky)::value>>(
          "conv1d_tc", grid, PP_THREADS, smem, stream, ta, tb, to, p);
    };
    const bool leaky = p.act == RAVE_ACT_LEAKY;
    return p.bias ? (leaky ? go(y, y) : go(y, n)) : (leaky ? go(n, y) : go(n, n));
  } else {
    // mask, skip and output boxes cover the tile's batch group; partner rows go one batch per box.  With fm_bh < 0
    // (the launch covers the fake half) the partner of batch b is batch b of the half stored right before dact_src.
    memset(&tp, 0, sizeof(tp));
    memset(&tr, 0, sizeof(tr));
    if (encode_rows_map<BN>(&tm, p.dact_src, p, p.BB)) return 1;
    if (p.fm_d && encode_rows_map<BN>(&tp, p.fm_bh > 0 ? p.dact_src : p.dact_src - p.fm_half, p, 1)) return 1;
    if (p.res_bf16 && encode_rows_map<BN>(&tr, p.res_bf16, p, p.BB)) return 1;
    const auto go = [&](auto fm, auto rs) {
      return launch_tc<conv_tc_pp_kernel<BN, BK, decltype(fm)::value, decltype(rs)::value>>(
          "conv1d_tc", grid, PP_THREADS, smem, stream, ta, tb, tm, tp, tr, to, p);
    };
    return p.fm_d ? (p.res_bf16 ? go(y, y) : go(y, n)) : (p.res_bf16 ? go(n, y) : go(n, n));
  }
}

template <int BN, int BK, bool X3>
static int launch(const CUtensorMap &ta, const CUtensorMap &tb, TcParams p, cudaStream_t stream) {
  using L = SmemLayout<BN, BK, X3>;
  plan_smem<BN, BK, X3>(p.K * p.num_kb, p);
  if (!p.out_act) p.stg = 0;
  CUtensorMap to;
  memset(&to, 0, sizeof(to));
  if (p.stg && encode_rows_map<BN>(&to, p.out_act, p, p.BB)) return 1;
  return launch_tc<conv_tc_kernel<BN, BK, X3>>("conv1d_tc", persistent_grid(p.n_lt * p.n_bg * p.n_nt), NUM_THREADS,
                                               p.bar_off + L::FIXED, stream, ta, tb, to, p);
}

// The split-operand (x3) instantiations live in their own translation unit (conv_tc_x3.cu includes this file with
// RAVE_TC_X3_UNIT defined) so that the two sets of kernels compile in parallel.
int conv_tc_dispatch_x3(int BK, int BN, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t s);
#ifdef RAVE_TC_X3_UNIT
int conv_tc_dispatch_x3(int BK, int BN, const CUtensorMap &ta, const CUtensorMap &tb, const TcParams &p, cudaStream_t s) {
  return visit_tile(BK, BN, [&](auto bk, auto bn) {
    return launch<decltype(bn)::value, decltype(bk)::value, true>(ta, tb, p, s);
  });
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

// Which kernel instance rave_conv1d_tc_fwd runs for a shape (writing out_act): BLOCK_N | BLOCK_K << 12 |
// (accumulator buffers - 1) << 24 | staged output << 25 | ring stages << 26; 0 = none.
extern "C" int rave_conv1d_tc_plan(int B, int Cin, int Cout, int Lout, int K) {
  using namespace rave::tc;
  const TcGeometry g = tc_geometry(B, Cin, Cout, Lout);
  if (!g.BK || !g.BN) return 0;
  TcParams q;
  visit_tile(g.BK, g.BN, [&](auto bk, auto bn) {
    plan_smem<decltype(bn)::value, decltype(bk)::value, false>(K * g.num_kb, q);
    return 0;
  });
  return g.BN | (g.BK << 12) | (q.nacc - 1) << 24 | q.stg << 25 | q.stages << 26;
}

// Ring stages of the ping-pong kernel for an input-gradient launch of this shape (LeakyReLU' mask, bf16 output only;
// fm: with the feature-matching partner rows, res_bf16: with the gradient skip); 0 = the launch runs conv_tc_kernel.
extern "C" int rave_conv1d_tc_pp_stages(int B, int Cin, int Cout, int Lout, int K, int fm, int res_bf16) {
  using namespace rave::tc;
  const TcGeometry g = tc_geometry(B, Cin, Cout, Lout);
  if (!g.BK || !g.BN) return 0;
  const int nops = 1 + (fm ? 1 : 0) + (res_bf16 ? 1 : 0);
  return visit_tile(g.BK, g.BN, [&](auto bk, auto bn) {
    return pp_stages<decltype(bn)::value, decltype(bk)::value, false>(nops);
  });
}

// Ring stages of the ping-pong kernel for a forward launch of this shape (bias and / or LeakyReLU, bf16 output only);
// 0 = the launch runs conv_tc_kernel.
extern "C" int rave_conv1d_tc_pp_fwd_stages(int B, int Cin, int Cout, int Lout, int K) {
  using namespace rave::tc;
  const TcGeometry g = tc_geometry(B, Cin, Cout, Lout);
  if (!g.BK || !g.BN) return 0;
  return visit_tile(g.BK, g.BN, [&](auto bk, auto bn) {
    return pp_fwd_stages<decltype(bn)::value, decltype(bk)::value>(K * g.num_kb);
  });
}

// Ring stages of the wide kernel (128 x 192 tiles, two MMA warpgroups per tile) for a forward launch of this shape (bias
// and / or LeakyReLU, bf16 output only); 0 = the launch does not run it.  A launch the wide kernel takes runs neither
// conv_tc_kernel nor the ping-pong kernel, whatever rave_conv1d_tc_plan and rave_conv1d_tc_pp_fwd_stages report for it.
extern "C" int rave_conv1d_tc_wide_stages(int B, int Cin, int Cout, int Lout, int K) {
  using namespace rave::tc;
  const TcGeometry g = tc_geometry(B, Cin, Cout, Lout);
  if (!g.BK || !g.BN) return 0;
  return wide_stages(Cin, Cout, K);
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
  RAVE_CHECK_ARG(get_encode_fn(), "conv1d_tc: cuTensorMapEncodeTiled not available");

  const TcGeometry g = tc_geometry(B, Cin, Cout, Lout);
  RAVE_CHECK_ARG(g.BN > 0, "conv1d_tc: no BLOCK_N for Cout=%d", Cout);
  // input-gradient launches (LeakyReLU' mask, optional feature-matching term and gradient skip, bf16 out only) and
  // forward launches (bias and / or LeakyReLU, bf16 out only): the ping-pong kernel where pp_stages / pp_fwd_stages
  // give it the launch; long-k forward launches with Cout % 192 == 0 the wide kernel (wide_stages)
  const bool bf16_only = out_act && !res && !res_act && !out_f32;
  const bool pp_dgrad = bf16_only && dact_src && !bias && act == RAVE_ACT_NONE;
  const bool pp_fwd = bf16_only && !dact_src && !res_bf16 && !fm_d;
  const int wide = !x3 && pp_fwd ? wide_stages(Cin, Cout, K) : 0;
  const int BK = wide ? wide_block_k(Cin) : g.BK, BN = wide ? WIDE_N : g.BN;
  // 256-byte L2 promotion over-fetches when a TMA row is a 64-byte (or shorter) span of a 192-byte channel row
  // (measured on the Cin = 96 layers: 209.6 -> 184.7 us); neutral to slightly positive for 128-byte spans.
  const CUtensorMapL2promotion promo = BK == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
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
  p.act_ld = x3 ? 2 * Cout : Cout;
  p.act_cs = act_cs > 0 ? act_cs : Cout;
  RAVE_CHECK_ARG(!x3 || (Cout % p.act_cs == 0 && p.act_cs % 16 == 0),
                 "conv1d_tc(x3): %d channels per position do not tile the %d-column rows in 16-column chunks", p.act_cs,
                 Cout);
  RAVE_CHECK_ARG(!x3 || !res_act || p.act_cs == Cout, "conv1d_tc(x3): res_act needs one position per row");
  p.BL = g.BL; p.BB = g.BB; p.n_lt = g.n_lt; p.n_bg = g.n_bg;
  p.n_nt = Cout / BN;
  p.num_kb = ceil_div(Cin, BK);

  // A: channel-last activations viewed as (c, phase, l/stride, b)
  CUtensorMap ta, tb;
  {
    const cuuint64_t ca = (cuuint64_t)Cin * (x3 ? 2 : 1);       // channels per activation row ([hi | lo] in x3 mode)
    const cuuint64_t dims[4] = {ca, (cuuint64_t)stride, (cuuint64_t)ceil_div(Lin, stride), (cuuint64_t)B};
    const cuuint64_t strides[3] = {ca * 2, ca * 2 * stride, ca * 2 * in_pitch};
    const cuuint32_t box[4] = {(cuuint32_t)BK, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    const CUresult r = encode_bf16_map(&ta, 4, xa, dims, strides, box, swizzle_enum(BK * 2), promo);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "conv1d_tc: tensor map A encode failed (%d)", (int)r);
  }
  {
    const cuuint64_t dims[2] = {(cuuint64_t)Cin, (cuuint64_t)K * Cout * (x3 ? 2 : 1)};
    const cuuint64_t strides[1] = {(cuuint64_t)Cin * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    const CUresult r = encode_bf16_map(&tb, 2, wt, dims, strides, box, swizzle_enum(BK * 2), promo);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "conv1d_tc: tensor map B encode failed (%d)", (int)r);
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (x3) return conv_tc_dispatch_x3(BK, BN, ta, tb, p, s);
  if (wide) return BK == 64 ? launch_wide<64>(ta, tb, p, wide, s) : launch_wide<32>(ta, tb, p, wide, s);
  const int nops = 1 + (fm_d ? 1 : 0) + (res_bf16 ? 1 : 0);
  return visit_tile(BK, BN, [&](auto bk, auto bn) {
    constexpr int BK_ = decltype(bk)::value, BN_ = decltype(bn)::value;
    if constexpr (pp_built<BN_, BK_, false>) {
      const int stages = pp_dgrad ? pp_stages<BN_, BK_, false>(nops) : 0;
      if (stages) return launch_pp<BN_, BK_, false>(ta, tb, p, stages, s);
    }
    if constexpr (pp_built<BN_, BK_, true>) {
      const int stages = pp_fwd ? pp_fwd_stages<BN_, BK_>(K * g.num_kb) : 0;
      if (stages) return launch_pp<BN_, BK_, true>(ta, tb, p, stages, s);
    }
    return launch<BN_, BK_, false>(ta, tb, p, s);
  });
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
// slice of the rows (split-K) and writes its partial tile to its own slice of dWt[splits][K][Cm][Cn] (no atomics);
// tapmajor_to_weight_kernel adds the slices in slice order.
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

  // tile / slice owned by this CTA.  The slice is the slowest index: the CTAs of one slice stream the same P and Q rows
  // (every tap, m-tile and n-tile of those rows) and run side by side, so each row comes from HBM about once and the
  // other tiles find it in L2.  With the slice fastest, a slice's tiles fell into different waves and every wave
  // re-read the rows.
  const int tiles = p.K * p.n_mt * p.n_nt;
  const int split = blockIdx.x / tiles;
  int t = blockIdx.x % tiles;
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
      const TapOrigin o = tap_origin(k, p.dil, p.pad_l, p.stride);
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
            tma_load_4d(sb + s * WG_SLAB, &tmap_q, &full_bar[stage], n0 + 64 * s, o.ph, l0 + o.j, b0);
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    } else if (warp < 4) {
      // MMA warpgroup: bf16 x bf16 -> fp32, A and B both MN-major (transposed operands); M half h = P slab h
      const uint32_t smem_base = smem_u32(smem);
      float d[2][BLOCK_N / 2];
      int stage = 0, prev = 0;        // prev: stage of the group still in flight (as in conv_tc_kernel)
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
        wgmma_wait<1>();                                         // the group of chunk c - 1 has completed
        if (c > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs<BLOCK_N / 2>(d[0]);
      wgmma_fence_regs<BLOCK_N / 2>(d[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
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

// one CTA per (tap, m-tile, n-tile, split)
template <int BN>
static int launch_wg(const CUtensorMap &tp, const CUtensorMap &tq, const WgParams &p, cudaStream_t stream) {
  return launch_tc<wgrad_tc_kernel<BN>>("wgrad_tc", p.K * p.n_mt * p.n_nt * p.splits, NUM_THREADS, WgSmem<BN>::TOTAL,
                                        stream, tp, tq, p);
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

// Tile rave_conv1d_tc_wgrad runs for a shape: BLOCK_N | BLOCK_M << 8 | ring stages << 16; the launch has
// K * splits * ceil(Cm / BLOCK_M) * ceil(Cn / BLOCK_N) CTAs (one tile each).
extern "C" int rave_conv1d_tc_wgrad_plan(int B, int Cm, int Lp, int Cn, int K) {
  using namespace rave::tc;
  int BL, n_lt, n_bg, n_mt, BN, n_nt, splits;
  wg_geometry(B, Cm, Lp, Cn, K, &BL, &n_lt, &n_bg, &n_mt, &BN, &n_nt, &splits);
  const int stages = BN == 64 ? WgSmem<64>::STAGES : WgSmem<128>::STAGES;
  return BN | 128 << 8 | stages << 16;
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
  RAVE_CHECK_ARG(get_encode_fn(), "wgrad_tc: cuTensorMapEncodeTiled not available");
  cudaStream_t s = (cudaStream_t)stream;

  WgParams p;
  p.B = B; p.Cm = Cm; p.Lp = Lp; p.Cn = Cn; p.Lq = Lq; p.K = K; p.stride = stride; p.dil = dil; p.pad_l = pad_l;
  p.dwt = dwt;
  p.dbias = dbias;
  int BN;
  wg_geometry(B, Cm, Lp, Cn, K, &p.BL, &p.n_lt, &p.n_bg, &p.n_mt, &BN, &p.n_nt, &p.splits);
  p.BB = WG_ROWS / p.BL;

  CUtensorMap tp, tq;
  const cuuint32_t box[4] = {64, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
  {
    const cuuint64_t dims[4] = {(cuuint64_t)Cm, 1, (cuuint64_t)Lp, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2 * p_pitch};
    const CUresult r = encode_bf16_map(&tp, 4, P, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_tc: tensor map P encode failed (%d)", (int)r);
  }
  {
    const cuuint64_t dims[4] = {(cuuint64_t)Cn, (cuuint64_t)stride, (cuuint64_t)ceil_div(Lq, stride), (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)Cn * 2, (cuuint64_t)Cn * 2 * stride, (cuuint64_t)Cn * 2 * q_pitch};
    const CUresult r = encode_bf16_map(&tq, 4, Q, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
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
