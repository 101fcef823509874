// Multi-tap weight gradient on wgmma (sm_90a):
//
//     dWt[k][m][n] = sum_{(b,l)} P[b][l][m] * Q[b][l*stride + k*dil - pad_l][n]          for ALL taps k of a group at once
//
// The per-tap kernel (conv_tc.cu: wgrad_tc_kernel) gives every tap its own CTA: each one streams the P rows (the output
// gradient) and its own shifted Q rows (the saved operand) from L2 -- K times the bytes of one pass.  Here a CTA owns a
// (128 x BN) tile of dW for a GROUP of taps (as many as its accumulator registers hold):
//
//   * the P tile [64 rows x 128 channels] is loaded ONCE per 64-row chunk and feeds every tap's MMAs;
//   * taps that read the same phase of Q (row = (l + j) * stride + ph) share ONE haloed Q tile: rows l0 + jmin ...
//     l0 + 63 + jmax of that phase.  Both operands are MN-major (the reduction runs over tile rows), so tap j is the same
//     tile with the descriptor's start address moved down (j - jmin) rows of 128 bytes: the 128-byte swizzle is a
//     function of the absolute shared-memory address (TMA wrote it that way), no copy, no re-layout;
//   * every tap has its own fp32 accumulator tile in the MMA warpgroup's registers (taps x BN <= 128 per thread).
//
// K = 15 / stride 4 in the row-widened form the engine uses (4 unit-stride taps over 4x wider rows): P 16 KB + Q 17 KB
// per 4 x 256 MMA clocks = 33 B/clk instead of 4 x 40 KB per the same work.  Split-K over row slices as before: every
// slice writes its own partial tile (no atomics), the weight-norm backward sums them in order.  The tap-group 0 / n-tile 0
// CTAs also reduce the P tiles over rows (bias gradient).
// Reference: autograd of F.conv1d / F.conv_transpose1d (weight gradient) at rave/blocks.py:96-108, 538-592, 637-692,
// rave/discriminator.py:99-111.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace rave {
namespace tc {

constexpr int WM_THREADS = 288;          // warps 0-3: MMA warpgroup (+ result store), warp 4: TMA producer, warps 5-8: column sums
constexpr int WM_ACC = 128;              // accumulator registers per MMA thread: taps x BLOCK_N
constexpr int WM_MAXT = 8;               // taps per CTA
constexpr int WM_ROWS = 64;              // reduction rows per pipeline stage
constexpr int WM_PSLAB = WM_ROWS * 128;  // [64 rows][64 ch] bf16
constexpr int WM_QROWS = 80;             // rows of a haloed Q slab: 64 + at most 16 halo rows (all batch segments)
constexpr int WM_QSLAB = WM_QROWS * 128;

struct WmParams {
  int B, Cm, Lp, Cn, Lq, K, stride, dil, pad_l;
  int BL, BB, n_lt, n_bg;      // row chunk = BB batches x BL rows (BL * BB == 64, BL >= 16)
  int n_mt, n_nt, splits;
  int tpg, n_groups;           // taps per group, tap groups (each CTA: one group)
  int halo;                    // extra rows every Q box carries (max over the tiles)
  int stages, stage_bytes;
  float *dwt;                  // [splits][K][Cm][Cn]
  float *dbias;
  float *dbias_part;           // [splits][n_mt * 128] per-slice partial bias gradients (see dbias_sum_kernel)
  // per tap: Q tile (index within its group) and row shift inside that tile; per group: first tile, tile count;
  // per tile: phase and first row offset j
  unsigned char tap_tile[32], tap_shift[32];
  unsigned char group_tile0[33];
  unsigned char tile_ph[40];
  signed char tile_j[40];
};

template <int BLOCK_N>
__global__ void __launch_bounds__(WM_THREADS, 1)
wgrad_mt_kernel(const __grid_constant__ CUtensorMap tmap_p, const __grid_constant__ CUtensorMap tmap_q,
                const WmParams p) {
  constexpr int NS = (BLOCK_N + 63) / 64;
  constexpr int MAXT = WM_ACC / BLOCK_N;               // taps per CTA this instance can hold
  constexpr int MAX_STAGES = 8;
  static_assert(BLOCK_N % 64 == 0 && MAXT >= 1, "MN-major B operand: whole 64-channel slabs");
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int bar_off = p.stages * p.stage_bytes;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + bar_off);
  uint64_t *empty_bar = full_bar + MAX_STAGES;
  float *cs_scratch = reinterpret_cast<float *>(smem + bar_off + 256);          // [8][128] fp32

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // tile / slice / tap group owned by this CTA
  const int split = blockIdx.x % p.splits;
  int t = blockIdx.x / p.splits;
  const int nt = t % p.n_nt; t /= p.n_nt;
  const int mt = t % p.n_mt; t /= p.n_mt;
  const int grp = t;
  const int k0 = grp * p.tpg;
  const int nk = min(p.tpg, p.K - k0);
  const int tile0 = p.group_tile0[grp], n_tiles = p.group_tile0[grp + 1] - tile0;
  const int m0 = mt * 128, n0 = nt * BLOCK_N;
  const int n_chunks = p.n_lt * p.n_bg;
  const int per = (n_chunks + p.splits - 1) / p.splits;
  const int ch_begin = split * per;
  const int ch_end = min(n_chunks, ch_begin + per);
  const int my_chunks = max(0, ch_end - ch_begin);
  const bool do_cs = p.dbias != nullptr && grp == 0 && nt == 0;
  const int qrows = p.BL + p.halo;                     // rows per batch segment of a Q box

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_p);
    tma_prefetch_desc(&tmap_q);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], do_cs ? 8 : 4);     // the 4 MMA warps (+ the 4 column-sum warps)
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();      // dependents may begin their prologue ...
  griddep_wait();                   // ... and this kernel touches global memory only after its predecessors are done

  if (my_chunks > 0) {
    if (warp == 4) {
      // =========================== TMA producer ===========================
      const uint32_t tx = 2 * WM_PSLAB + (uint32_t)n_tiles * NS * (uint32_t)(qrows * p.BB * 128);
      int stage = 0;
      uint32_t phase = 0;
      for (int ch = ch_begin; ch < ch_end; ++ch) {
        const int lt = ch % p.n_lt, bg = ch / p.n_lt;
        const int l0 = lt * p.BL, b0 = bg * p.BB;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t *sa = smem + stage * p.stage_bytes;
        uint8_t *sq = sa + 2 * WM_PSLAB;
        if (elect_one()) {
          mbar_arrive_expect_tx(&full_bar[stage], tx);
          tma_load_4d(sa, &tmap_p, &full_bar[stage], m0, 0, l0, b0);
          tma_load_4d(sa + WM_PSLAB, &tmap_p, &full_bar[stage], m0 + 64, 0, l0, b0);
          for (int ti = 0; ti < n_tiles; ++ti) {
            const int ph = p.tile_ph[tile0 + ti], j = p.tile_j[tile0 + ti];
#pragma unroll
            for (int s = 0; s < NS; ++s)
              tma_load_4d(sq + (ti * NS + s) * WM_QSLAB, &tmap_q, &full_bar[stage], n0 + 64 * s, ph, l0 + j, b0);
          }
        }
        __syncwarp();
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    } else if (warp < 4) {
      // =========================== MMA warpgroup ===========================
      // bf16 x bf16 -> fp32, A and B both MN-major (transposed operands); M half h = P slab h
      const uint32_t smem_base = smem_u32(smem);
      float d[MAXT][2][BLOCK_N / 2];
      int stage = 0;
      uint32_t phase = 0;
      for (int c = 0; c < my_chunks; ++c) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_base + stage * p.stage_bytes;
        const uint32_t sq = sa + 2 * WM_PSLAB;
        wgmma_fence();
#pragma unroll
        for (int i = 0; i < MAXT; ++i) {
          if (i < nk) {
            const uint32_t qt = sq + (uint32_t)p.tap_tile[k0 + i] * NS * WM_QSLAB;
            const int shift = p.tap_shift[k0 + i];
#pragma unroll
            for (int kk = 0; kk < WM_ROWS / 16; ++kk) {
              // reduction rows 16 kk .. 16 kk + 15 = batch segment (16 kk) / BL, rows (16 kk) % BL ...: the same rows of
              // the Q box, `shift` rows further down
              const int r = 16 * kk;
              const int qrow = (r / p.BL) * qrows + (r % p.BL) + shift;
              const uint64_t bdesc = make_mnmajor_desc(qt + qrow * 128, WM_QSLAB);
#pragma unroll
              for (int h = 0; h < 2; ++h)
                Wgmma<BLOCK_N, 1, 1>::mma(d[i][h], make_mnmajor_desc(sa + h * WM_PSLAB + r * 128, WM_PSLAB), bdesc,
                                          (c > 0 || kk > 0) ? 1u : 0u);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < MAXT; ++i) {
          wgmma_fence_regs<BLOCK_N / 2>(d[i][0]);
          wgmma_fence_regs<BLOCK_N / 2>(d[i][1]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
#pragma unroll
      for (int i = 0; i < MAXT; ++i)
        if (i < nk)
          store_wgrad_tile<BLOCK_N>(d[i], p.dwt + ((size_t)split * p.K + (k0 + i)) * p.Cm * p.Cn, m0, n0, p.Cm, p.Cn);
    } else if (do_cs) {
      // bias gradient: column sums of the P tiles while the tensor core consumes them (as in wgrad_tc_kernel)
      const int te = (warp - 5) * 32 + lane;
      const int cg = te & 15, rg = te >> 4;
      const uint32_t col = (uint32_t)(cg >> 3) * WM_PSLAB + (uint32_t)(((cg & 7) ^ rg) << 4);
      float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      int stage = 0;
      uint32_t phase = 0;
      for (int c = 0; c < my_chunks; ++c) {
        mbar_wait(&full_bar[stage], phase);
        const uint8_t *sa = smem + stage * p.stage_bytes + col;
#pragma unroll
        for (int i = 0; i < WM_ROWS / 8; ++i) {
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
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) cs_scratch[rg * 128 + cg * 8 + j] = cs[j];
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float tsum = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) tsum += cs_scratch[r * 128 + te];
      p.dbias_part[(size_t)split * p.n_mt * 128 + m0 + te] = tsum;
    }
  } else if (do_cs && warp >= 5) {
    // empty slice: no rows, zero partial bias gradient
    p.dbias_part[(size_t)split * p.n_mt * 128 + m0 + (warp - 5) * 32 + lane] = 0.f;
  } else if (warp < 4) {
    // empty slice (more splits than row chunks): this CTA still owns its partial tiles -> zeros
    const int m = m0 + threadIdx.x;
    if (m < p.Cm) {
      for (int i = 0; i < nk; ++i) {
        float *dst = p.dwt + (((size_t)split * p.K + (k0 + i)) * p.Cm + m) * p.Cn + n0;
        for (int c = 0; c < BLOCK_N; ++c)
          if (n0 + c < p.Cn) dst[c] = 0.f;
      }
    }
  }
}

typedef CUresult (*EncodeTiledFnW)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                   const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFnW wm_encode_fn() {
  static EncodeTiledFnW fn = nullptr;
  if (!fn) {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFnW)ptr;
  }
  return fn;
}

// N tile and taps per CTA from the shape alone (the split count the caller allocates for must not depend on stride /
// dilation / padding): whole 64-channel slabs of Q, as many taps as share one P tile within the WM_ACC accumulator
// registers of an MMA thread
static void wm_tile(int Cn, int K, int *BN, int *tpg) {
  const int bn = (Cn <= 64 || K > 1) ? 64 : 128;
  int t = WM_ACC / bn;
  if (t > K) t = K;
  *BN = bn;
  *tpg = t;
}

static void wm_geometry(int B, int Cm, int Lp, int Cn, int K, int *BL, int *n_lt, int *n_bg, int *n_mt, int *BN,
                        int *n_nt, int *tpg, int *n_groups, int *splits) {
  int bl = WM_ROWS;
  while (bl > Lp && bl > 16) bl >>= 1;
  *BL = bl;
  *n_lt = ceil_div(Lp, bl);
  *n_bg = ceil_div(B, WM_ROWS / bl);
  *n_mt = ceil_div(Cm, 128);
  wm_tile(Cn, K, BN, tpg);
  *n_nt = ceil_div(Cn, *BN);
  *n_groups = ceil_div(K, *tpg);
  const int tiles = (*n_groups) * (*n_mt) * (*n_nt);
  const int n_chunks = (*n_lt) * (*n_bg);
  int s = ceil_div(tiles >= 66 ? 132 : 2 * 132, tiles);
  if (s > 32) s = 32;
  if (s > n_chunks / 4) s = n_chunks / 4;      // at least 4 chunks of 64 rows per slice
  if (s > n_chunks) s = n_chunks;
  if (s < 1) s = 1;
  *splits = s;
}

template <int BN>
static int launch_wm(const CUtensorMap &tp, const CUtensorMap &tq, const WmParams &p, int smem_bytes,
                     cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_mt_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("wgrad_mt: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return 2;
    }
    attr = true;
  }
  const int grid = p.n_groups * p.n_mt * p.n_nt * p.splits;
  launch_pdl(wgrad_mt_kernel<BN>, dim3(grid), dim3(WM_THREADS), smem_bytes, stream, tp, tq, p);
  RAVE_CHECK_LAUNCH("wgrad_mt");
  return 0;
}

}  // namespace tc
}  // namespace rave

// Fills the tap / tile tables, halo, stage size and depth of `p` (geometry fields already set); false when the tap
// pattern does not fit one CTA's haloed tiles (the per-tap kernel then takes the layer).
static bool wm_build_tiles(rave::tc::WmParams &p, int BN, int K, int stride, int dil, int pad_l) {
  using namespace rave::tc;
  // ---- Q tiles of every tap group: taps of one phase whose row offsets j stay within the halo budget share a tile
  const int halo_budget = 16 / p.BB;
  int n_tiles_total = 0, max_tiles = 0, halo = 0;
  for (int g = 0; g < p.n_groups; ++g) {
    p.group_tile0[g] = (unsigned char)n_tiles_total;
    const int ka = g * p.tpg, kb = (ka + p.tpg < K) ? ka + p.tpg : K;
    int t_ph[WM_MAXT], t_jmin[WM_MAXT], t_jmax[WM_MAXT], nt_g = 0;
    for (int k = ka; k < kb; ++k) {
      const int off = k * dil - pad_l;
      int j = off / stride, ph = off - j * stride;
      if (ph < 0) { ph += stride; j -= 1; }
      int hit = -1;
      for (int t = 0; t < nt_g; ++t) {
        if (t_ph[t] != ph) continue;
        const int lo = j < t_jmin[t] ? j : t_jmin[t], hi = j > t_jmax[t] ? j : t_jmax[t];
        if (hi - lo <= halo_budget) { hit = t; t_jmin[t] = lo; t_jmax[t] = hi; break; }
      }
      if (hit < 0) { hit = nt_g; t_ph[nt_g] = ph; t_jmin[nt_g] = t_jmax[nt_g] = j; ++nt_g; }
      p.tap_tile[k] = (unsigned char)hit;
      p.tap_shift[k] = 0;      // filled below (jmin may still move)
    }
    for (int k = ka; k < kb; ++k) {
      const int off = k * dil - pad_l;
      int j = off / stride, ph = off - j * stride;
      if (ph < 0) { ph += stride; j -= 1; }
      p.tap_shift[k] = (unsigned char)(j - t_jmin[p.tap_tile[k]]);
    }
    for (int t = 0; t < nt_g; ++t) {
      if (n_tiles_total >= 40) return false;
      p.tile_ph[n_tiles_total] = (unsigned char)t_ph[t];
      if (t_jmin[t] < -128 || t_jmin[t] > 127) return false;
      p.tile_j[n_tiles_total] = (signed char)t_jmin[t];
      if (t_jmax[t] - t_jmin[t] > halo) halo = t_jmax[t] - t_jmin[t];
      ++n_tiles_total;
    }
    if (nt_g > max_tiles) max_tiles = nt_g;
  }
  p.group_tile0[p.n_groups] = (unsigned char)n_tiles_total;
  p.halo = halo;
  if ((p.BL + halo) * p.BB > WM_QROWS) return false;
  const int NS = (BN + 63) / 64;
  p.stage_bytes = 2 * WM_PSLAB + max_tiles * NS * WM_QSLAB;
  p.stages = (227 * 1024 - 1024 - 256 - 4096) / p.stage_bytes;
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 2) return false;            // too many distinct Q tiles for one CTA: per-tap kernel
  return true;
}

// 1 when the multi-tap kernel takes this shape (rows per batch >= 16 ... see the checks below); the per-tap kernel
// covers the rest.  RAVE_WG_MT=0 disables it.
extern "C" int rave_conv1d_tc_wgrad_mt_supported(int B, int Cm, int Lp, int Cn, int K) {
  // OPT-IN (RAVE_WG_MT=1): numerically right (tests/test_gpu_tc.py runs it), but the tensor core re-reads the P tile
  // from shared memory for every tap and at most two taps fit the register accumulators, so it is not the default.
  const char *e = getenv("RAVE_WG_MT");
  if (!(e && e[0] == '1')) return 0;
  if (K < 1 || K > 32 || Cm % 8 || Cn % 8) return 0;
  if (Lp < 16) return 0;                 // 16-row MMA slices must not straddle batch segments
  return 1;
}

extern "C" int rave_conv1d_tc_wgrad_mt_splits(int B, int Cm, int Lp, int Cn, int K) {
  int BL, n_lt, n_bg, n_mt, BN, n_nt, tpg, n_groups, splits;
  rave::tc::wm_geometry(B, Cm, Lp, Cn, K, &BL, &n_lt, &n_bg, &n_mt, &BN, &n_nt, &tpg, &n_groups, &splits);
  return splits;
}

// Split count of the multi-tap kernel for this layer (the caller allocates dwt[splits][K][Cm][Cn]), or 0 when the
// per-tap kernel (rave_conv1d_tc_wgrad, with ITS split count) must run it.
extern "C" int rave_conv1d_tc_wgrad_mt_plan(int B, int Cm, int Lp, int Cn, int K, int stride, int dil, int pad_l) {
  using namespace rave::tc;
  if (!rave_conv1d_tc_wgrad_mt_supported(B, Cm, Lp, Cn, K)) return 0;
  WmParams p;
  memset(&p, 0, sizeof(p));
  int BN;
  wm_geometry(B, Cm, Lp, Cn, K, &p.BL, &p.n_lt, &p.n_bg, &p.n_mt, &BN, &p.n_nt, &p.tpg, &p.n_groups, &p.splits);
  p.BB = WM_ROWS / p.BL;
  p.K = K;
  if (!wm_build_tiles(p, BN, K, stride, dil, pad_l)) return 0;
  return p.splits;
}

// Same contract as rave_conv1d_tc_wgrad (include/rave_b200.h), for layers rave_conv1d_tc_wgrad_mt_plan accepts.
extern "C" int rave_conv1d_tc_wgrad_mt(const void *P, const void *Q, float *dwt, float *dbias, int B, int Cm, int Lp,
                                       int p_pitch, int Cn, int Lq, int q_pitch, int K, int stride, int dil, int pad_l,
                                       void *stream) {
  using namespace rave;
  using namespace rave::tc;
  RAVE_CHECK_ARG(P && Q && dwt, "wgrad_mt: null pointer");
  RAVE_CHECK_ARG(rave_conv1d_tc_wgrad_mt_supported(B, Cm, Lp, Cn, K), "wgrad_mt: unsupported shape");
  if (p_pitch <= 0) p_pitch = Lp;
  if (q_pitch <= 0) q_pitch = Lq;
  RAVE_CHECK_ARG(q_pitch >= ceil_div(Lq, stride) * stride,
                 "wgrad_mt: Q pitch %d < Lq %d rounded up to the stride %d (slack rows must be zero)", q_pitch, Lq, stride);
  EncodeTiledFnW enc = wm_encode_fn();
  RAVE_CHECK_ARG(enc, "wgrad_mt: cuTensorMapEncodeTiled not available");

  WmParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.Cm = Cm; p.Lp = Lp; p.Cn = Cn; p.Lq = Lq; p.K = K; p.stride = stride; p.dil = dil; p.pad_l = pad_l;
  p.dwt = dwt; p.dbias = dbias;
  int BN;
  wm_geometry(B, Cm, Lp, Cn, K, &p.BL, &p.n_lt, &p.n_bg, &p.n_mt, &BN, &p.n_nt, &p.tpg, &p.n_groups, &p.splits);
  p.BB = WM_ROWS / p.BL;
  if (!wm_build_tiles(p, BN, K, stride, dil, pad_l)) {
    set_error("wgrad_mt: tap pattern does not fit (call rave_conv1d_tc_wgrad_mt_plan first)");
    return 1;
  }
  const int smem_bytes = p.stages * p.stage_bytes + 256 + 4096 + 1024;

  CUtensorMap tp, tq;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cm, 1, (cuuint64_t)Lp, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2, (cuuint64_t)Cm * 2 * p_pitch};
    cuuint32_t box[4] = {64, 1, (cuuint32_t)p.BL, (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(P), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_mt: tensor map P encode failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cn, (cuuint64_t)stride, (cuuint64_t)ceil_div(Lq, stride), (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cn * 2, (cuuint64_t)Cn * 2 * stride, (cuuint64_t)Cn * 2 * q_pitch};
    cuuint32_t box[4] = {64, 1, (cuuint32_t)(p.BL + p.halo), (cuuint32_t)p.BB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tq, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(Q), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RAVE_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_mt: tensor map Q encode failed (%d)", (int)r);
  }
  cudaStream_t s = (cudaStream_t)stream;
  p.dbias_part = nullptr;
  if (dbias && cudaMallocAsync((void **)&p.dbias_part, sizeof(float) * p.splits * p.n_mt * 128, s) != cudaSuccess) {
    set_error("wgrad_mt: cudaMallocAsync of the bias-gradient partials failed");
    return 2;
  }
  int rc = 1;
  switch (BN) {
    case 64: rc = launch_wm<64>(tp, tq, p, smem_bytes, s); break;
    case 128: rc = launch_wm<128>(tp, tq, p, smem_bytes, s); break;
    default: set_error("wgrad_mt: no kernel for BLOCK_N=%d", BN);
  }
  if (dbias) {
    if (rc == 0) {
      dbias_sum_kernel<<<ceil_div(Cm, 256), 256, 0, s>>>(p.dbias_part, dbias, p.splits, p.n_mt * 128, Cm);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) {
        set_error("wgrad_mt: dbias_sum launch failed: %s", cudaGetErrorString(e));
        rc = 2;
      } else {
        count_launch();
      }
    }
    cudaFreeAsync(p.dbias_part, s);
  }
  return rc;
}
