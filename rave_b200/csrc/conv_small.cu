// Small-channel kernels of the discriminators: layers that are NOT GEMM shaped and are bound by the
// HBM traffic of their channel-last feature maps, written as direct CUDA-core kernels with coalesced
// channel-contiguous access (north star: "warp shuffles for the small channel reductions, tensor
// cores only where the contraction is genuinely dense").
//
//   * first conv of every ConvNet (Cin = 1): nn.Conv1d(1, C, 15, 4, 7) of the multi-scale and
//     nn.Conv2d(1, C, (5,1), (4,1), (2,0)) of the multi-period discriminator, rave/discriminator.py:99-111
//     (the folded period axis is extra batch) -- forward and weight gradient;
//   * the feature-matching statistics of rave/model.py:360-368 (core.mean_difference, L1 / relative,
//     rave/core.py:236-252) evaluated directly on the engine's bf16 operand stream a = LeakyReLU(h):
//     S_diff = sum |h_real - h_fake|, S_abs = sum |h_real|, and the gradient of those two sums.
#include "common.cuh"

namespace rave {

__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t *>(&h);
}

// ---------------------------------------------------------------------------------------------
// out[r][l][co] = bias[co] + sum_k w[co][k] * x[r][l*stride + k - pad_l]      (x zero outside [0,Lin))
// x: [R][x_pitch] fp32; outputs channel-last [R][out_pitch][Cout]: fp32 stream and/or bf16 act(out)
// one thread = one output row position x 8 consecutive channels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv_c1_fwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                   float *__restrict__ out_f32, __nv_bfloat16 *__restrict__ out_act, int R, int x_pitch, int Lin,
                   int Cout, int Lout, int out_pitch, int K, int stride, int pad_l, int act, float slope) {
  extern __shared__ float sw[];   // [K][Cout] + bias[Cout]
  float *sb = sw + K * Cout;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int k = i / Cout, co = i - k * Cout;
    sw[i] = w[co * K + k];
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sb[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int chunks = Cout >> 3;
  const int r = blockIdx.y;                         // one batch row per grid.y
  const float *xr = x + (size_t)r * x_pitch;
  const int per_row = Lout * chunks;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_row; i += gridDim.x * blockDim.x) {
    const int l = i / chunks;
    const int c8 = (i - l * chunks) * 8;
    const int base = l * stride - pad_l;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = sb[c8 + j];
    for (int k = 0; k < K; ++k) {
      const int pos = base + k;
      const float xv = (pos >= 0 && pos < Lin) ? __ldg(xr + pos) : 0.f;
      const float4 w0 = *reinterpret_cast<const float4 *>(sw + k * Cout + c8);
      const float4 w1 = *reinterpret_cast<const float4 *>(sw + k * Cout + c8 + 4);
      acc[0] = fmaf(xv, w0.x, acc[0]); acc[1] = fmaf(xv, w0.y, acc[1]);
      acc[2] = fmaf(xv, w0.z, acc[2]); acc[3] = fmaf(xv, w0.w, acc[3]);
      acc[4] = fmaf(xv, w1.x, acc[4]); acc[5] = fmaf(xv, w1.y, acc[5]);
      acc[6] = fmaf(xv, w1.z, acc[6]); acc[7] = fmaf(xv, w1.w, acc[7]);
    }
    const size_t o = ((size_t)r * out_pitch + l) * Cout + c8;
    if (out_f32) {
      float4 *o4 = reinterpret_cast<float4 *>(out_f32 + o);
      o4[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      o4[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    if (out_act) {
      if (act == RAVE_ACT_LEAKY) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = acc[j] > 0.f ? acc[j] : acc[j] * slope;
      }
      *reinterpret_cast<uint4 *>(out_act + o) = make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]),
                                                          pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// dwt[cta][k][co] = sum_{(r,l) in the CTA's slice} g[r][l][co] * x[r][l*stride + k - pad_l]
// g: bf16 channel-last [R][g_pitch][Cg] (only the first Cout channels are read).
// block = Cout x NL threads (thread = one channel, NL row lanes); K <= 16 accumulators per thread.
// ---------------------------------------------------------------------------------------------
constexpr int C1_MAXK = 16;

// grid (slices_per_row, R): each CTA reduces a contiguous slice of positions of ONE batch row.
// thread = 2 adjacent channels x one of NL position lanes, 4 positions in flight per thread.
__global__ void __launch_bounds__(256)
conv_c1_wgrad_kernel(const __nv_bfloat16 *__restrict__ g, const float *__restrict__ x, float *__restrict__ dwt,
                     int R, int x_pitch, int Lin, int Cout, int Cg, int Lout, int g_pitch, int K, int stride,
                     int pad_l, int NL, const BlockSum bs) {
  extern __shared__ float red[];   // [NL][K][Cout]
  const int half = Cout >> 1;
  const int c2 = (threadIdx.x % half) * 2;
  const int lane = threadIdx.x / half;
  const int r = blockIdx.y;
  float acc0[C1_MAXK], acc1[C1_MAXK];
#pragma unroll
  for (int k = 0; k < C1_MAXK; ++k) { acc0[k] = 0.f; acc1[k] = 0.f; }
  const int per = (Lout + gridDim.x - 1) / gridDim.x;
  const int begin = blockIdx.x * per;
  const int end = min(Lout, begin + per);
  const float *xr = x + (size_t)r * x_pitch;
  const __nv_bfloat16 *gr = g + (size_t)r * g_pitch * Cg + c2;
  if (lane < NL) {
    for (int l0 = begin + lane; l0 < end; l0 += 4 * NL) {
      uint32_t gw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int l = l0 + u * NL;
        gw[u] = (l < end) ? *reinterpret_cast<const uint32_t *>(gr + (size_t)l * Cg) : 0u;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int l = l0 + u * NL;
        if (l >= end) break;
        const float g0 = bf16_lo(gw[u]), g1 = bf16_hi(gw[u]);
        const int base = l * stride - pad_l;
#pragma unroll
        for (int k = 0; k < C1_MAXK; ++k) {
          if (k < K) {
            const int pos = base + k;
            const float xv = (pos >= 0 && pos < Lin) ? __ldg(xr + pos) : 0.f;
            acc0[k] = fmaf(g0, xv, acc0[k]);
            acc1[k] = fmaf(g1, xv, acc1[k]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < C1_MAXK; ++k)
      if (k < K) {
        red[((size_t)lane * K + k) * Cout + c2] = acc0[k];
        red[((size_t)lane * K + k) * Cout + c2 + 1] = acc1[k];
      }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    float s = 0.f;
    for (int ln = 0; ln < NL; ++ln) s += red[(size_t)ln * K * Cout + i];
    block_sum_put(bs, i, s);
  }
  block_sum_finish(bs, dwt);               // [k][co]  (== [1][K][C0p=Cout][C1p=1]), pre-zeroed
}

// ---------------------------------------------------------------------------------------------
// input gradient of the first conv:  dx[r][t] = sum_k sum_co g[r][(t + pad - k)/stride][co] w[co][k]
// (terms with a non-integer / out-of-range row dropped).  One CTA = 256 consecutive samples of one
// batch row: stage 1 computes P[l][k] = <g[r][l][:], w[:][k]> for the ~256/stride + K/stride rows that
// touch the tile, stage 2 gathers.  g: bf16 channel-last [R][g_pitch][Cg].
// ---------------------------------------------------------------------------------------------
constexpr int C1_DG_TILE = 256;

__global__ void __launch_bounds__(256)
conv_c1_dgrad_kernel(const __nv_bfloat16 *__restrict__ g, const float *__restrict__ w, float *__restrict__ dx,
                     int x_pitch, int Lin, int Cout, int Cg, int Lout, int g_pitch, int K, int stride, int pad_l) {
  extern __shared__ float sm[];                 // w [K][Cout]  |  P [rows][K]
  float *sw = sm;
  float *P = sm + K * Cout;
  const int r = blockIdx.y;
  const int t0 = blockIdx.x * C1_DG_TILE;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int k = i / Cout, co = i - k * Cout;
    sw[i] = w[co * K + k];
  }
  // rows l with l*stride + k - pad in [t0, t0 + TILE) for some k in [0, K)
  int lmin = (t0 + pad_l - (K - 1) + stride - 1) / stride;
  if (t0 + pad_l - (K - 1) < 0) lmin = 0;
  int lmax = (t0 + C1_DG_TILE - 1 + pad_l) / stride;
  if (lmax > Lout - 1) lmax = Lout - 1;
  const int nrows = lmax - lmin + 1;
  __syncthreads();
  // stage 1: one warp per row, lanes over channel pairs, shuffle-reduce; K dot products per row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int rr = warp; rr < nrows; rr += 8) {
    const __nv_bfloat16 *gp = g + ((size_t)r * g_pitch + (lmin + rr)) * Cg;
    float part[C1_MAXK];
#pragma unroll
    for (int k = 0; k < C1_MAXK; ++k) part[k] = 0.f;
    for (int c2 = lane * 2; c2 < Cout; c2 += 64) {
      const uint32_t gw = *reinterpret_cast<const uint32_t *>(gp + c2);
      const float g0 = bf16_lo(gw), g1 = bf16_hi(gw);
#pragma unroll
      for (int k = 0; k < C1_MAXK; ++k)
        if (k < K) part[k] = fmaf(g0, sw[k * Cout + c2], fmaf(g1, sw[k * Cout + c2 + 1], part[k]));
    }
#pragma unroll
    for (int k = 0; k < C1_MAXK; ++k) {
      if (k < K) {
        float v = part[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) P[rr * K + k] = v;
      }
    }
  }
  __syncthreads();
  // stage 2: gather
  const int t = t0 + threadIdx.x;
  if (t < Lin) {
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
      const int q = t + pad_l - k;
      if (q < 0) break;
      const int l = q / stride;
      if (l * stride == q && l >= lmin && l <= lmax) acc += P[(l - lmin) * K + k];
    }
    dx[(size_t)r * x_pitch + t] = acc;
  }
}

// column sums of a bf16 channel-last tensor: out[c] = sum_{r, l < L} g[r][l][c]   (conv bias gradient)
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const __nv_bfloat16 *__restrict__ g, float *__restrict__ out, int L, int pitch, int Cg, int C,
                   const BlockSum bs) {
  // grid (slices, R); block 256 = 32 position lanes x 8 channel groups; each thread strides channels
  __shared__ float red[8][33];
  const int r = blockIdx.y;
  const int per = (L + gridDim.x - 1) / gridDim.x;
  const int begin = blockIdx.x * per, end = min(L, begin + per);
  const int lane_l = threadIdx.x >> 5;      // 0..7 : position lane
  const int lane_c = threadIdx.x & 31;      // channel lane
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + lane_c;
    float s = 0.f;
    if (c < C)
      for (int l = begin + lane_l; l < end; l += 8) s += __bfloat162float(g[((size_t)r * pitch + l) * Cg + c]);
    red[lane_l][lane_c] = s;
    __syncthreads();
    if (lane_l == 0 && c < C) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += red[i][lane_c];
      block_sum_put(bs, c, t);
    }
    __syncthreads();
  }
  block_sum_finish(bs, out);
}

// ---------------------------------------------------------------------------------------------
// feature-matching statistics on a = LeakyReLU(h) (bf16, channel-last [2*Bh][pitch][C]); the first Bh
// batch entries are "real", the last Bh "fake" (rave/model.py:349-352 concatenates [x, y]).
// stats[0] += sum |h_r - h_f|, stats[1] += sum |h_r|   over l < L, c < C.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float unleaky(float a, float inv_slope) { return a > 0.f ? a : a * inv_slope; }
__device__ __forceinline__ void ldg256_nc(const void *p, uint32_t *r) {     // 32-byte aligned, read-only
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "l"(p));
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
               : "l"(reinterpret_cast<const uint8_t *>(p) + 16));
}

// grid (blocks per batch entry, Bh): a batch entry's valid rows [L][C] are one contiguous range, so the index is linear
// (no 64-bit divisions per element); two 32-byte row pieces per half in flight per thread.
__global__ void __launch_bounds__(256)
fm_stats_kernel(const __nv_bfloat16 *__restrict__ a, float *__restrict__ stats, int Bh, int L, int pitch, int C,
                float inv_slope, const BlockSum bs) {
  __shared__ float red0[8], red1[8];
  const long n_vec = (long)L * (C >> 4);                    // 16-channel vectors of one batch entry
  const size_t half = (size_t)Bh * pitch * C;
  const __nv_bfloat16 *ar = a + (size_t)blockIdx.y * pitch * C;
  const float2 inv2 = make_float2(inv_slope, inv_slope);
  float2 s0 = make_float2(0.f, 0.f), s1 = make_float2(0.f, 0.f);
  const long stride = (long)gridDim.x * 256;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n_vec; i += 2 * stride) {
    uint32_t rw[2][8], fw[2][8];
    const long i2 = i + stride;
    ldg256_nc(ar + i * 16, rw[0]);
    ldg256_nc(ar + i * 16 + half, fw[0]);
    const bool two = i2 < n_vec;
    if (two) {
      ldg256_nc(ar + i2 * 16, rw[1]);
      ldg256_nc(ar + i2 * 16 + half, fw[1]);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !two) break;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 r = make_float2(bf16_lo(rw[u][j]), bf16_hi(rw[u][j]));
        const float2 f = make_float2(bf16_lo(fw[u][j]), bf16_hi(fw[u][j]));
        const float2 rs = make_float2(r.x * inv2.x, r.y * inv2.y), fs = make_float2(f.x * inv2.x, f.y * inv2.y);
        // inverse LeakyReLU (1 / slope >= 1): h = min(a, a / slope)
        const float2 hr = make_float2(fminf(r.x, rs.x), fminf(r.y, rs.y));
        const float2 hf = make_float2(fminf(f.x, fs.x), fminf(f.y, fs.y));
        const float2 d = make_float2(hr.x - hf.x, hr.y - hf.y);
        s0 = make_float2(s0.x + fabsf(d.x), s0.y + fabsf(d.y));
        s1 = make_float2(s1.x + fabsf(hr.x), s1.y + fabsf(hr.y));
      }
    }
  }
  float t0 = s0.x + s0.y, t1 = s1.x + s1.y;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    t0 += __shfl_xor_sync(0xffffffffu, t0, o);
    t1 += __shfl_xor_sync(0xffffffffu, t1, o);
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red0[wid] = t0; red1[wid] = t1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float u0 = 0.f, u1 = 0.f;
    for (int i = 0; i < 8; ++i) { u0 += red0[i]; u1 += red1[i]; }
    block_sum_put(bs, 0, u0);
    block_sum_put(bs, 1, u1);
  }
  block_sum_finish(bs, stats);
}

// gradient of (d0 * S_diff + d1 * S_abs) with respect to h, written as the bf16 gradient stream:
//   real rows: d0 sgn(h_r - h_f) + d1 sgn(h_r);  fake rows: -d0 sgn(h_r - h_f);  slack rows (l >= L): 0
__global__ void __launch_bounds__(256)
fm_grad_kernel(const __nv_bfloat16 *__restrict__ a, const float *__restrict__ dstats,
               __nv_bfloat16 *__restrict__ gout, int Bh, int L, int pitch, int C, float inv_slope) {
  const float d0 = dstats[0], d1 = dstats[1];
  const int vecs = C >> 3;
  const long total = (long)Bh * pitch * vecs;
  const size_t half = (size_t)Bh * pitch * C;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int v = (int)(i % vecs);
    const long bl = i / vecs;
    const int l = (int)(bl % pitch);
    const int b = (int)(bl / pitch);
    const size_t o = ((size_t)b * pitch + l) * C + v * 8;
    uint32_t gr[4] = {0, 0, 0, 0}, gf[4] = {0, 0, 0, 0};
    if (l < L) {
      const uint4 r = *reinterpret_cast<const uint4 *>(a + o);
      const uint4 f = *reinterpret_cast<const uint4 *>(a + o + half);
      const uint32_t rw[4] = {r.x, r.y, r.z, r.w}, fw[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float o_r[2], o_f[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float ar = h ? bf16_hi(rw[j]) : bf16_lo(rw[j]);
          const float af = h ? bf16_hi(fw[j]) : bf16_lo(fw[j]);
          const float hr = unleaky(ar, inv_slope), hf = unleaky(af, inv_slope);
          const float sd = (hr > hf) ? 1.f : ((hr < hf) ? -1.f : 0.f);
          const float sr = (hr > 0.f) ? 1.f : ((hr < 0.f) ? -1.f : 0.f);
          o_r[h] = d0 * sd + d1 * sr;
          o_f[h] = -d0 * sd;
        }
        gr[j] = pack_bf16(o_r[0], o_r[1]);
        gf[j] = pack_bf16(o_f[0], o_f[1]);
      }
    }
    *reinterpret_cast<uint4 *>(gout + o) = make_uint4(gr[0], gr[1], gr[2], gr[3]);
    *reinterpret_cast<uint4 *>(gout + o + half) = make_uint4(gf[0], gf[1], gf[2], gf[3]);
  }
}

}  // namespace rave

extern "C" int rave_conv1d_c1_fwd(const float *x, const float *w, const float *bias, float *out_f32,
                                  void *out_act_bf16, int R, int x_pitch, int Lin, int Cout, int Lout,
                                  int out_pitch, int K, int stride, int pad_l, int act, float slope, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && w && (out_f32 || out_act_bf16), "conv1d_c1_fwd: null pointer");
  RAVE_CHECK_ARG(R > 0 && Lin > 0 && Lout > 0 && Cout > 0 && Cout % 8 == 0 && K > 0 && stride > 0,
                 "conv1d_c1_fwd: bad shape (Cout must be a multiple of 8)");
  RAVE_CHECK_ARG(act == RAVE_ACT_NONE || act == RAVE_ACT_LEAKY, "conv1d_c1_fwd: unsupported activation");
  RAVE_CHECK_ARG(R <= 65535, "conv1d_c1_fwd: too many rows");
  const int per_row = Lout * (Cout / 8);
  int bx = (per_row + 255) / 256;
  const int want = (132 * 16 + R - 1) / R;       // ~16 CTAs per SM in total
  if (bx > want) bx = want;
  if (bx < 1) bx = 1;
  const size_t smem = (size_t)(K + 1) * Cout * sizeof(float);
  conv_c1_fwd_kernel<<<dim3(bx, R), 256, smem, (cudaStream_t)stream>>>(
      x, w, bias, out_f32, (__nv_bfloat16 *)out_act_bf16, R, x_pitch, Lin, Cout, Lout, out_pitch, K, stride, pad_l,
      act, slope);
  RAVE_CHECK_LAUNCH("conv1d_c1_fwd");
  return 0;
}

static int c1_wgrad_slices(int R, int Lout) {
  int sl = (132 * 8 + R - 1) / R;                 // ~8 CTAs per SM in total
  const int max_sl = (Lout + 63) / 64;            // at least 64 positions per slice
  if (sl > max_sl) sl = max_sl;
  if (sl < 1) sl = 1;
  return sl;
}

extern "C" int rave_conv1d_c1_wgrad_splits(int R, int Lout) { return 1; }

extern "C" int rave_conv1d_c1_wgrad(const void *g_bf16, const float *x, float *dwt, int R, int x_pitch, int Lin,
                                    int Cout, int Cg, int Lout, int g_pitch, int K, int stride, int pad_l,
                                    void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(g_bf16 && x && dwt, "conv1d_c1_wgrad: null pointer");
  RAVE_CHECK_ARG(K > 0 && K <= C1_MAXK && Cout > 0 && Cout <= 512 && Cout % 2 == 0 && Cg >= Cout && Cg % 2 == 0,
                 "conv1d_c1_wgrad: bad shape");
  RAVE_CHECK_ARG(R <= 65535, "conv1d_c1_wgrad: too many rows");
  const int slices = c1_wgrad_slices(R, Lout);
  const int half = Cout / 2;
  int NL = 256 / half;
  if (NL < 1) NL = 1;
  const int threads = half * NL;
  const size_t smem = (size_t)NL * K * Cout * sizeof(float);
  RAVE_CHECK_ARG(smem <= 48 * 1024, "conv1d_c1_wgrad: reduction buffer too large");
  cudaMemsetAsync(dwt, 0, sizeof(float) * K * Cout, (cudaStream_t)stream);
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, (long)slices * R, K * Cout, (cudaStream_t)stream)) return rc;
  conv_c1_wgrad_kernel<<<dim3(slices, R), threads, smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)g_bf16, x, dwt, R, x_pitch, Lin, Cout, Cg, Lout, g_pitch, K, stride, pad_l, NL, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("conv1d_c1_wgrad");
  return 0;
}

extern "C" int rave_conv1d_c1_dgrad(const void *g_bf16, const float *w, float *dx, int R, int x_pitch, int Lin,
                                    int Cout, int Cg, int Lout, int g_pitch, int K, int stride, int pad_l,
                                    void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(g_bf16 && w && dx, "conv1d_c1_dgrad: null pointer");
  RAVE_CHECK_ARG(K > 0 && K <= C1_MAXK && Cout > 0 && Cout % 2 == 0 && Cg >= Cout && Cg % 2 == 0 && R <= 65535,
                 "conv1d_c1_dgrad: bad shape");
  const int max_rows = C1_DG_TILE / stride + (K - 1) / stride + 3;
  const size_t smem = ((size_t)K * Cout + (size_t)max_rows * K) * sizeof(float);
  RAVE_CHECK_ARG(smem <= 48 * 1024, "conv1d_c1_dgrad: shared memory");
  dim3 grid(ceil_div(Lin, C1_DG_TILE), R);
  conv_c1_dgrad_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>((const __nv_bfloat16 *)g_bf16, w, dx, x_pitch, Lin,
                                                                 Cout, Cg, Lout, g_pitch, K, stride, pad_l);
  RAVE_CHECK_LAUNCH("conv1d_c1_dgrad");
  return 0;
}

extern "C" int rave_colsum_bf16(const void *g_bf16, float *out, int R, int L, int pitch, int Cg, int C,
                                void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(g_bf16 && out && R > 0 && R <= 65535 && L > 0 && pitch >= L && C > 0 && Cg >= C,
                 "colsum_bf16: bad argument");
  cudaMemsetAsync(out, 0, sizeof(float) * C, (cudaStream_t)stream);
  int sl = (132 * 8 + R - 1) / R;
  const int max_sl = (L + 63) / 64;
  if (sl > max_sl) sl = max_sl;
  if (sl < 1) sl = 1;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, (long)sl * R, C, (cudaStream_t)stream)) return rc;
  colsum_bf16_kernel<<<dim3(sl, R), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)g_bf16, out, L, pitch, Cg, C, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("colsum_bf16");
  return 0;
}

extern "C" int rave_fm_stats(const void *a_bf16, float *stats, int Bh, int L, int pitch, int C, float slope,
                             void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(a_bf16 && stats && Bh > 0 && L > 0 && pitch >= L && C > 0 && C % 16 == 0 && slope > 0.f &&
                     ((uintptr_t)a_bf16 & 31) == 0,
                 "fm_stats: bad argument (C %% 16 == 0, 32-byte aligned operand)");
  RAVE_CHECK_ARG(Bh <= 65535, "fm_stats: %d batch entries per half > 65535", Bh);
  const long per_b = (long)L * (C / 16);
  long bx = (per_b + 511) / 512;                     // two vectors per thread and pass
  const long cap = (132L * 8 + Bh - 1) / Bh;         // ~8 blocks per SM over the whole grid
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, bx * Bh, 2, (cudaStream_t)stream)) return rc;
  fm_stats_kernel<<<dim3((unsigned)bx, (unsigned)Bh), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)a_bf16, stats,
                                                                                    Bh, L, pitch, C, 1.f / slope, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("fm_stats");
  return 0;
}

extern "C" int rave_fm_grad(const void *a_bf16, const float *dstats, void *gout_bf16, int Bh, int L, int pitch,
                            int C, float slope, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(a_bf16 && dstats && gout_bf16 && Bh > 0 && L > 0 && pitch >= L && C > 0 && C % 8 == 0 &&
                     slope > 0.f,
                 "fm_grad: bad argument");
  const long total = (long)Bh * pitch * (C / 8);
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  fm_grad_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)a_bf16, dstats,
                                                                (__nv_bfloat16 *)gout_bf16, Bh, L, pitch, C,
                                                                1.f / slope);
  RAVE_CHECK_LAUNCH("fm_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Discriminator score tail (rave/model.py:348-379 with core.hinge_gan / core.mean_difference): every scalar the
// training step derives from the score map s = last conv output (channel 0 of the channel-last fp32 tensor
// [2*Bh][pitch][C], real half first) comes from six sums, produced by one launch instead of ~40 ATen launches
// per ConvNet (and as many again in the backward):
//   stats[0] = sum |s_r - s_f|    stats[1] = sum |s_r|          (score as the last feature-matching term)
//   stats[2] = sum relu(1 - s_r)  stats[3] = sum relu(1 + s_f)  (hinge discriminator loss)
//   stats[4] = sum s_r            stats[5] = sum s_f            (adversarial loss, pred_real / pred_fake)
// score_grad_kernel is the gradient of sum_i d[i] * stats[i] with respect to s, written as the bf16 gradient
// stream of the last conv (other channels and slack rows zero).
// ---------------------------------------------------------------------------------------------
namespace rave {

__global__ void __launch_bounds__(256)
score_stats_kernel(const float *__restrict__ s, float *__restrict__ stats, int Bh, int L, int pitch, int C,
                   const BlockSum bs) {
  __shared__ float red[6][8];
  const long total = (long)Bh * L;
  const size_t half = (size_t)Bh * pitch * C;
  float a[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int l = (int)(i % L);
    const int b = (int)(i / L);
    const size_t o = ((size_t)b * pitch + l) * C;
    const float sr = s[o], sf = s[o + half];
    a[0] += fabsf(sr - sf);
    a[1] += fabsf(sr);
    a[2] += fmaxf(1.f - sr, 0.f);
    a[3] += fmaxf(1.f + sf, 0.f);
    a[4] += sr;
    a[5] += sf;
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a[j] += __shfl_xor_sync(0xffffffffu, a[j], o);
    if (lane == 0) red[j][wid] = a[j];
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
    block_sum_put(bs, threadIdx.x, t);
  }
  block_sum_finish(bs, stats);
}

__global__ void __launch_bounds__(256)
score_grad_kernel(const float *__restrict__ s, const float *__restrict__ d, __nv_bfloat16 *__restrict__ gout,
                  int Bh, int L, int pitch, int C) {
  const float d0 = d[0], d1 = d[1], d2 = d[2], d3 = d[3], d4 = d[4], d5 = d[5];
  const long total = (long)Bh * pitch;
  const size_t half = (size_t)Bh * pitch * C;
  const int vecs = C >> 3;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int l = (int)(i % pitch);
    const size_t o = (size_t)i * C;
    float gr = 0.f, gf = 0.f;
    if (l < L) {
      const float sr = s[o], sf = s[o + half];
      const float sd = sr > sf ? 1.f : (sr < sf ? -1.f : 0.f);
      const float sa = sr > 0.f ? 1.f : (sr < 0.f ? -1.f : 0.f);
      gr = d0 * sd + d1 * sa - (sr < 1.f ? d2 : 0.f) + d4;
      gf = -d0 * sd + (sf > -1.f ? d3 : 0.f) + d5;
    }
    uint4 *pr = reinterpret_cast<uint4 *>(gout + o);
    uint4 *pf = reinterpret_cast<uint4 *>(gout + o + half);
    pr[0] = make_uint4(pack_bf16(gr, 0.f), 0u, 0u, 0u);
    pf[0] = make_uint4(pack_bf16(gf, 0.f), 0u, 0u, 0u);
    for (int v = 1; v < vecs; ++v) {
      pr[v] = make_uint4(0u, 0u, 0u, 0u);
      pf[v] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

}  // namespace rave

extern "C" int rave_score_stats(const float *score, float *stats, int Bh, int L, int pitch, int C, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(score && stats && Bh > 0 && L > 0 && pitch >= L && C > 0, "score_stats: bad argument");
  long blocks = ((long)Bh * L + 255) / 256;
  if (blocks > 132 * 4) blocks = 132 * 4;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 6, (cudaStream_t)stream)) return rc;
  score_stats_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(score, stats, Bh, L, pitch, C, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("score_stats");
  return 0;
}

extern "C" int rave_score_grad(const float *score, const float *dstats, void *gout_bf16, int Bh, int L, int pitch,
                               int C, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(score && dstats && gout_bf16 && Bh > 0 && L > 0 && pitch >= L && C > 0 && C % 8 == 0,
                 "score_grad: bad argument");
  long blocks = ((long)Bh * pitch + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  score_grad_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(score, dstats, (__nv_bfloat16 *)gout_bf16, Bh, L,
                                                                   pitch, C);
  RAVE_CHECK_LAUNCH("score_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Cin = 1 first layer on the tensor-core kernels: the K (<= 16) taps become 16 "channels" of a tiny
// im2col, X[r][l][k] = bf16(x[r][l*stride + k - pad_l]) (33 MB for the 64 x 16384-row MSD input), so
//   forward : conv_tc (Cin = 16, one tap)            out[r][l][co] = sum_k X[r][l][k] w[co][k]
//   wgrad   : wgrad_tc (P = g, Q = X, one tap)       dw[co][k]     = sum_{r,l} g[r][l][co] X[r][l][k]
//   dgrad   : conv_tc (Cin = Cout, Cout = 16) -> P[r][l][k] = <g[r][l][:], w[:][k]>, then the gather below
//             dx[r][t] = sum_k P[r][(t + pad - k)/stride][k]
// ---------------------------------------------------------------------------------------------
namespace rave {

// Source addressing shared by the im2col and its adjoint: the R chain rows are derived from a signal tensor
// src[Bs][src_pitch] (src_len valid samples) WITHOUT materialising them:
//   row r = b*period + w,  position i  ->  (1/pool) * sum_{j<pool} src[b][(i*pool + j)*period + w]
// period > 1: MultiPeriodDiscriminator.fold (zero padding to a multiple of the period, rave/discriminator.py:187-195);
// pool > 1: the avg_pool1d(2) chain of MultiScaleDiscriminator (rave/discriminator.py:150-171, pool = 2^scale).
__device__ __forceinline__ float c1_src_value(const float *__restrict__ xb, int i, int w, int period, int pool,
                                              int src_len) {
  float v = 0.f;
  for (int j = 0; j < pool; ++j) {
    const long e = ((long)i * pool + j) * period + w;
    if (e < src_len) v += __ldg(xb + e);
  }
  return pool > 1 ? v / (float)pool : v;
}

// Writes one X row: column j = c*K + k (the [c][k] order of weight.reshape(Cout, Cin*K)), zero from cin*K to W (cin = 0:
// an all-zero slack row).  The running (c, k) pair replaces a division per column; `val(c, k)` is the source value of
// channel c at tap k.  Each 16-byte group is stored as soon as it is packed: only 4 words stay live (at W = 32 the
// whole row held in registers cut the staged kernel's occupancy to a third).
template <int W, typename F>
__device__ __forceinline__ void write_cin_row(__nv_bfloat16 *dst_row, int cin, int K, F val) {
  uint4 *dst = reinterpret_cast<uint4 *>(dst_row);
  int c = 0, k = 0;
#pragma unroll
  for (int q = 0; q < W / 8; ++q) {
    uint32_t wd[4];
#pragma unroll
    for (int j2 = 0; j2 < 4; ++j2) {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        v[h] = c < cin ? val(c, k) : 0.f;
        if (++k == K) {
          k = 0;
          ++c;
        }
      }
      wd[j2] = pack_bf16(v[0], v[1]);
    }
    dst[q] = make_uint4(wd[0], wd[1], wd[2], wd[3]);
  }
}

// Per-thread variant, only for shapes whose staged tile (below) exceeds 96 KB of shared memory (large periods).
// grid (ceil(pitch/256), R), block 256: one thread = one position = one 2W-byte row of X (W/8 16-byte stores);
// the K source positions of neighbouring threads overlap (K > stride), so the strided reads hit in L1
template <int W>
__global__ void __launch_bounds__(256)
im2col_cin_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ X, int cin, int src_pitch, int src_len,
                  int Lin, int Lout, int out_pitch, int K, int stride, int pad_l, int period, int pool) {
  const int r = blockIdx.y;
  const int l = blockIdx.x * 256 + threadIdx.x;
  if (l >= out_pitch) return;
  const int b = r / period, w = r - b * period;
  const float *xb = x + (size_t)b * cin * src_pitch;
  const int p0 = l * stride - pad_l;
  write_cin_row<W>(X + ((size_t)r * out_pitch + l) * W, l < Lout ? cin : 0, K, [&](int c, int k) {
    const int p = p0 + k;
    return (p >= 0 && p < Lin) ? c1_src_value(xb + (size_t)c * src_pitch, p, w, period, pool, src_len) : 0.f;
  });
}

// Staged variant (every tile up to 96 KB): the per-thread gather above issues K strided loads per output row and
// channel -- a warp access touches 32 addresses (stride * period) floats apart, 8-44 sectors for 128 useful bytes, and
// the L1 wavefront queue, not HBM, set its pace (40 us for a 33 MB operand).  Here one CTA serves IC_NL output
// positions of ALL `period` rows of one source batch entry: the contiguous source span of each channel is read once,
// coalesced, and de-interleaved into shared memory (one padded line per channel and fold row (c, w); the index skew
// i + i/32 makes the stride-`stride` tap reads conflict-free for stride 1, 2, 4); every thread then assembles 2W-byte
// rows from shared memory and stores them back to back.
constexpr int IC_NL = 128;
__device__ __forceinline__ int ic_skew(int i) { return i + (i >> 5); }

template <int W>
__global__ void __launch_bounds__(256, 4)   // >= 32 warps per SM: the W = 32 instance otherwise takes 98 registers
im2col_cin_staged_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ X, int cin, int src_pitch,
                         int src_len, int Lin, int Lout, int out_pitch, int K, int stride, int pad_l, int period,
                         int pool, int line) {
  extern __shared__ float sm[];                      // [cin][period][line]
  const int b = blockIdx.y;
  const int l0 = blockIdx.x * IC_NL;
  const int p_lo = l0 * stride - pad_l;
  const int n_p = (IC_NL - 1) * stride + K;
  for (int c = 0; c < cin; ++c) {
    const float *xb = x + ((size_t)b * cin + c) * src_pitch;
    float *smc = sm + (size_t)c * period * line;
    if (period > 1) {                                // fold: element (p, w) lives at p * period + w
      const long e_lo = (long)p_lo * period;
      for (int q = threadIdx.x; q < n_p * period; q += blockDim.x) {
        const int pp = q / period, w = q - pp * period;
        const int pos = p_lo + pp;
        const long e = e_lo + q;
        smc[w * line + ic_skew(pp)] = (pos >= 0 && pos < Lin && e < src_len) ? __ldg(xb + e) : 0.f;
      }
    } else {                                         // average pooling: position p = mean of `pool` consecutive samples
      for (int pp = threadIdx.x; pp < n_p; pp += blockDim.x) {
        const int pos = p_lo + pp;
        smc[ic_skew(pp)] = (pos >= 0 && pos < Lin) ? c1_src_value(xb, pos, 0, 1, pool, src_len) : 0.f;
      }
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < IC_NL * period; idx += blockDim.x) {
    const int w = idx / IC_NL, ll = idx - w * IC_NL;
    const int l = l0 + ll;
    if (l >= out_pitch) continue;
    const float *row = sm + w * line;
    const int q0 = ll * stride, cs = period * line;
    write_cin_row<W>(X + ((size_t)(b * period + w) * out_pitch + l) * W, l < Lout ? cin : 0, K,
                     [&](int c, int k) { return row[c * cs + ic_skew(q0 + k)]; });
  }
}

// dsrc[b][c][(t*pool + j)*period + w] += (1/pool) * sum_k P[r][(t + pad - k)/stride][c*K + k]; P fp32 channel-last
// [R][p_pitch][W].  Every source element is touched by at most one (r, t, j) thread: plain read-modify-write, launches
// are stream-ordered.
template <int W>
__global__ void __launch_bounds__(256)
gather_cin_kernel(const float *__restrict__ P, float *__restrict__ dx, int cin, int src_pitch, int src_len, int Lin,
                  int Lout, int p_pitch, int K, int stride, int pad_l, int period, int pool) {
  const int r = blockIdx.y;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Lin) return;
  const float *Pr = P + (size_t)r * p_pitch * W;
  // taps k = k0 + m stride hit output rows l0 - m: ONE integer division per thread (the loop used to divide twice per
  // tap by the run-time stride: ~125 of the thread's ~150 instructions)
  const int l0 = (t + pad_l) / stride;
  const int k0 = (t + pad_l) - l0 * stride;
  const int b = r / period, w = r - b * period;
  for (int c = 0; c < cin; ++c) {
    float acc = 0.f;
    for (int k = k0, l = l0; k < K && l >= 0; k += stride, --l)
      if (l < Lout) acc += __ldg(Pr + (size_t)l * W + c * K + k);
    float *db = dx + ((size_t)b * cin + c) * src_pitch;
    if (pool > 1) acc /= (float)pool;
    for (int j = 0; j < pool; ++j) {
      const long e = ((long)t * pool + j) * period + w;
      if (e < src_len) db[e] += acc;
    }
  }
}

}  // namespace rave

static inline int ic_skew_host(int i) { return i + (i >> 5); }

template <int W>
static int im2col_cin_launch(const float *x, void *X_bf16, int R, int cin, int src_pitch, int src_len, int Lin,
                             int Lout, int out_pitch, int K, int stride, int pad_l, int period, int pool,
                             void *stream) {
  using namespace rave;
  const int n_p = (IC_NL - 1) * stride + K;
  const int line = (ic_skew_host(n_p - 1) + 1) | 1;    // odd pitch: the de-interleaving stores spread over the banks
  const size_t smem = (size_t)cin * period * line * sizeof(float);
  if (stride >= 1 && smem <= 96 * 1024) {
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(im2col_cin_staged_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      attr = true;
    }
    dim3 grid(ceil_div(out_pitch, IC_NL), R / period);
    // period 1: 128 rows per CTA -> 128 threads (one row each); folds: 128 * period rows over 256 threads
    im2col_cin_staged_kernel<W><<<grid, period == 1 ? 128 : 256, smem, (cudaStream_t)stream>>>(
        x, (__nv_bfloat16 *)X_bf16, cin, src_pitch, src_len, Lin, Lout, out_pitch, K, stride, pad_l, period, pool, line);
    RAVE_CHECK_LAUNCH("im2col_cin_staged");
    return 0;
  }
  dim3 grid(ceil_div(out_pitch, 256), R);
  im2col_cin_kernel<W><<<grid, 256, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16 *)X_bf16, cin, src_pitch, src_len,
                                                               Lin, Lout, out_pitch, K, stride, pad_l, period, pool);
  RAVE_CHECK_LAUNCH("im2col_cin");
  return 0;
}

extern "C" int rave_im2col_cin(const float *x, void *X_bf16, int R, int cin, int src_pitch, int src_len, int Lin,
                               int Lout, int out_pitch, int W, int K, int stride, int pad_l, int period, int pool,
                               void *stream) {
  RAVE_CHECK_ARG(x && X_bf16 && R > 0 && R <= 65535 && cin >= 1 && K > 0 && (W == 16 || W == 32) && cin * K <= W &&
                     out_pitch >= Lout && period >= 1 && pool >= 1 && (period == 1 || pool == 1) && R % period == 0,
                 "im2col_cin: bad argument");
  if (W == 16)
    return im2col_cin_launch<16>(x, X_bf16, R, cin, src_pitch, src_len, Lin, Lout, out_pitch, K, stride, pad_l, period,
                                 pool, stream);
  return im2col_cin_launch<32>(x, X_bf16, R, cin, src_pitch, src_len, Lin, Lout, out_pitch, K, stride, pad_l, period,
                               pool, stream);
}

extern "C" int rave_gather_cin(const float *P, float *dsrc, int R, int cin, int src_pitch, int src_len, int Lin,
                               int Lout, int p_pitch, int W, int K, int stride, int pad_l, int period, int pool,
                               void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(P && dsrc && R > 0 && R <= 65535 && cin >= 1 && K > 0 && (W == 16 || W == 32) && cin * K <= W &&
                     p_pitch >= Lout && period >= 1 && pool >= 1 && (period == 1 || pool == 1) && R % period == 0,
                 "gather_cin: bad argument");
  dim3 grid(ceil_div(Lin, 256), R);
  if (W == 16)
    gather_cin_kernel<16><<<grid, 256, 0, (cudaStream_t)stream>>>(P, dsrc, cin, src_pitch, src_len, Lin, Lout, p_pitch,
                                                                  K, stride, pad_l, period, pool);
  else
    gather_cin_kernel<32><<<grid, 256, 0, (cudaStream_t)stream>>>(P, dsrc, cin, src_pitch, src_len, Lin, Lout, p_pitch,
                                                                  K, stride, pad_l, period, pool);
  RAVE_CHECK_LAUNCH("gather_cin");
  return 0;
}

extern "C" int rave_im2col_c1(const float *x, void *X_bf16, int R, int src_pitch, int src_len, int Lin, int Lout,
                              int out_pitch, int K, int stride, int pad_l, int period, int pool, void *stream) {
  return rave_im2col_cin(x, X_bf16, R, 1, src_pitch, src_len, Lin, Lout, out_pitch, 16, K, stride, pad_l, period,
                         pool, stream);
}
extern "C" int rave_gather_c1(const float *P, float *dsrc, int R, int src_pitch, int src_len, int Lin, int Lout,
                              int p_pitch, int K, int stride, int pad_l, int period, int pool, void *stream) {
  return rave_gather_cin(P, dsrc, R, 1, src_pitch, src_len, Lin, Lout, p_pitch, 16, K, stride, pad_l, period, pool,
                         stream);
}

// ---------------------------------------------------------------------------------------------
// L1 feature-matching statistics of two fp32 tensors (core.mean_difference, norm = L1: rave/core.py:236-252, called
// once per discriminator feature at rave/model.py:356-361): stats[0] += sum |t - v|, stats[1] += sum |t| in ONE pass
// (the torch form is sub, abs, mean, abs, mean, div + their backward: ~16 launches per feature, 108 features in a v3
// step), and the gradient of d0 * stats[0] + d1 * stats[1] in one pass.
// ---------------------------------------------------------------------------------------------
namespace rave {

__global__ void __launch_bounds__(256)
l1_stats_f32_kernel(const float *__restrict__ t, const float *__restrict__ v, float *__restrict__ stats, long n,
                    int vec, const BlockSum bs) {
  __shared__ float red0[8], red1[8];
  float s0 = 0.f, s1 = 0.f;
  if (!vec) {           // operands not 16-byte aligned (odd-sized slices): scalar pass
    for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
      s0 += fabsf(t[i] - v[i]);
      s1 += fabsf(t[i]);
    }
    n = 0;
  }
  const long n4 = n >> 2;
  const float4 *t4 = reinterpret_cast<const float4 *>(t), *v4 = reinterpret_cast<const float4 *>(v);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n4; i += (long)gridDim.x * 256) {
    const float4 a = __ldg(t4 + i), b = __ldg(v4 + i);
    s0 += fabsf(a.x - b.x) + fabsf(a.y - b.y) + fabsf(a.z - b.z) + fabsf(a.w - b.w);
    s1 += fabsf(a.x) + fabsf(a.y) + fabsf(a.z) + fabsf(a.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long i = (n4 << 2) + threadIdx.x;
    s0 += fabsf(t[i] - v[i]);
    s1 += fabsf(t[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red0[wid] = s0; red1[wid] = s1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float u0 = 0.f, u1 = 0.f;
    for (int i = 0; i < 8; ++i) { u0 += red0[i]; u1 += red1[i]; }
    block_sum_put(bs, 0, u0);
    block_sum_put(bs, 1, u1);
  }
  block_sum_finish(bs, stats);
}

__device__ __forceinline__ float sgnf(float x) { return (x > 0.f ? 1.f : 0.f) - (x < 0.f ? 1.f : 0.f); }

// gt = d0 sgn(t - v) + d1 sgn(t) (or null), gv = -d0 sgn(t - v) (or null)
__global__ void __launch_bounds__(256)
l1_grad_f32_kernel(const float *__restrict__ t, const float *__restrict__ v, const float *__restrict__ d,
                   float *__restrict__ gt, float *__restrict__ gv, long n) {
  const float d0 = d[0], d1 = d[1];
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float a = t[i], b = v[i];
    const float s = d0 * sgnf(a - b);
    if (gt) gt[i] = s + d1 * sgnf(a);
    if (gv) gv[i] = -s;
  }
}

}  // namespace rave

extern "C" int rave_l1_stats_f32(const float *t, const float *v, float *stats, long n, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(t && v && stats && n > 0, "l1_stats: bad argument");
  const int vec = ((((uintptr_t)t | (uintptr_t)v) & 15) == 0) ? 1 : 0;
  long blocks = ((vec ? (n >> 2) : n) + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 2, (cudaStream_t)stream)) return rc;
  l1_stats_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(t, v, stats, n, vec, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("l1_stats");
  return 0;
}

extern "C" int rave_l1_grad_f32(const float *t, const float *v, const float *d, float *gt, float *gv, long n,
                                void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(t && v && d && (gt || gv) && n > 0, "l1_grad: bad argument");
  long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  l1_grad_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(t, v, d, gt, gv, n);
  RAVE_CHECK_LAUNCH("l1_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Operand of a (kt, kf) Conv2d run as a conv along frequency (descript_discriminator.DiscConv2d, MRD of
// rave/descript_discriminator.py:118-184): x [B][C][T][F] fp32 -> channel-last bf16 rows
//   out[(b, t)][f][dt * C + c] = x[b][c][t + dt - pt][f]      (zero outside 0 <= t + dt - pt < T, f >= F, channel >= kt C)
// i.e. the kt time-shifted copies of the input channels side by side, and its adjoint.  One pass each instead of
// pad + stack + permute + reshape + pad + cast + contiguous (and their autograd).
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int TS_CP_MAX = 128;
constexpr int TS_PITCH = TS_CP_MAX + 8;      // bf16 elements per staged row (16-byte multiple)

// block = one (b, t) row x 32 frequency positions: loads coalesced along f (x is [.., T, F]), the [32][Cp] output block
// is contiguous in memory and leaves as 16-byte vectors
__global__ void __launch_bounds__(256)
time_stack_cl_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ out, int C, int T, int F, int Fp, int Cp,
                     int kt, int pt) {
  __shared__ __align__(16) __nv_bfloat16 tile[32][TS_PITCH];
  const int f0 = blockIdx.x * 32, t = blockIdx.y, b = blockIdx.z;
  const int fl = threadIdx.x & 31, cl = threadIdx.x >> 5;
  const int f = f0 + fl;
  const int nch = kt * C;
  for (int ch = cl; ch < Cp; ch += 8) {
    float v = 0.f;
    if (ch < nch && f < F) {
      const int dt = ch / C, c = ch - dt * C;
      const int ts = t + dt - pt;
      if (ts >= 0 && ts < T) v = __ldg(x + (((size_t)b * C + c) * T + ts) * F + f);
    }
    tile[fl][ch] = __float2bfloat16(v);
  }
  __syncthreads();
  const int rows = min(32, Fp - f0);
  const int vpr = Cp >> 3;                                      // 16-byte vectors per row (Cp % 8 == 0)
  uint4 *dst = reinterpret_cast<uint4 *>(out + (((size_t)b * T + t) * Fp + f0) * Cp);
  for (int i = threadIdx.x; i < rows * vpr; i += 256) {
    const int r = i / vpr, q = i - r * vpr;
    dst[i] = *reinterpret_cast<const uint4 *>(&tile[r][q * 8]);
  }
}

// adjoint: gx[b][c][tp][f] = sum_dt g[(b, tp + pt - dt)][f][dt * C + c]; the kt [32][Cp] blocks are staged through shared
// memory as 16-byte vectors, the result leaves coalesced along f
__global__ void __launch_bounds__(256)
time_stack_cl_bwd_kernel(const __nv_bfloat16 *__restrict__ g, float *__restrict__ gx, int C, int T, int F, int Fp,
                         int Cp, int kt, int pt) {
  __shared__ __align__(16) __nv_bfloat16 tile[32][TS_PITCH];
  const int f0 = blockIdx.x * 32, tp = blockIdx.y, b = blockIdx.z;
  const int fl = threadIdx.x & 31, cl = threadIdx.x >> 5;
  const int rows = min(32, Fp - f0);
  const int vpr = Cp >> 3;
  float acc[TS_CP_MAX / 2 / 8];                                 // channels cl, cl + 8, ... of this thread's f
#pragma unroll
  for (int j = 0; j < TS_CP_MAX / 2 / 8; ++j) acc[j] = 0.f;
  for (int dt = 0; dt < kt; ++dt) {
    const int t = tp + pt - dt;             // the output row whose slot dt read x[.., tp, ..]
    if (t >= 0 && t < T) {                  // (uniform per block)
      const uint4 *src = reinterpret_cast<const uint4 *>(g + (((size_t)b * T + t) * Fp + f0) * Cp);
      for (int i = threadIdx.x; i < rows * vpr; i += 256) {
        const int r = i / vpr, q = i - r * vpr;
        *reinterpret_cast<uint4 *>(&tile[r][q * 8]) = src[i];
      }
      __syncthreads();
      if (fl < rows) {
#pragma unroll
        for (int j = 0; j < TS_CP_MAX / 2 / 8; ++j) {
          const int c = cl + 8 * j;
          if (c < C) acc[j] += __bfloat162float(tile[fl][dt * C + c]);
        }
      }
      __syncthreads();
    }
  }
  if (f0 + fl < F) {
#pragma unroll
    for (int j = 0; j < TS_CP_MAX / 2 / 8; ++j) {
      const int c = cl + 8 * j;
      if (c < C) gx[(((size_t)b * C + c) * T + tp) * F + f0 + fl] = acc[j];
    }
  }
}

// Channel-last source (the MRD keeps its activations channel-last between layers: the conv output [(b, t)][f][c] IS the
// next layer's [b][t][f][c]): x[b][t][f][c] fp32 with element strides (sb, st), f-stride C, channels contiguous.
//   out[(b, t)][f][dt * C + c] = x[b][t + dt * dil - pt][f][c]
// (dil > 1: the time dilation of the EncodecConvNet convs of the multi-scale spectral discriminator).
// One thread = 8 output channels = one 16-byte store; with C % 8 == 0 its 8 sources are two 16-byte loads of one tap.
__global__ void __launch_bounds__(256)
time_stack_nhwc_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ out, long sb, long st, int C, int T, int F,
                       int Fp, int Cp, int kt, int pt, int dil, long total_vec, int vec) {
  const int vpr = Cp >> 3;
  const int nch = kt * C;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total_vec; i += (long)gridDim.x * 256) {
    const int cv = (int)(i % vpr);
    const long r = i / vpr;
    const int f = (int)(r % Fp);
    const long bt = r / Fp;
    const int t = (int)(bt % T);
    const long b = bt / T;
    const int ch0 = cv * 8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    if (f < F && ch0 < nch) {
      if (vec) {
        const int dt = ch0 / C, c = ch0 - dt * C;
        const int ts = t + dt * dil - pt;
        if (ts >= 0 && ts < T) {
          const float4 *p = reinterpret_cast<const float4 *>(x + b * sb + ts * st + (long)f * C + c);
          const float4 a0 = __ldg(p), a1 = __ldg(p + 1);
          v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w;
          v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int ch = ch0 + j;
          if (ch < nch) {
            const int dt = ch / C, c = ch - dt * C;
            const int ts = t + dt * dil - pt;
            if (ts >= 0 && ts < T) v[j] = __ldg(x + b * sb + ts * st + (long)f * C + c);
          }
        }
      }
    }
    uint4 o;
    __nv_bfloat162 h;
    h = __floats2bfloat162_rn(v[0], v[1]); o.x = *reinterpret_cast<uint32_t *>(&h);
    h = __floats2bfloat162_rn(v[2], v[3]); o.y = *reinterpret_cast<uint32_t *>(&h);
    h = __floats2bfloat162_rn(v[4], v[5]); o.z = *reinterpret_cast<uint32_t *>(&h);
    h = __floats2bfloat162_rn(v[6], v[7]); o.w = *reinterpret_cast<uint32_t *>(&h);
    reinterpret_cast<uint4 *>(out)[i] = o;
  }
}

// adjoint into a contiguous [B][T][F][C] fp32 gradient: gx[b][tp][f][c] = sum_dt g[(b, tp + pt - dt * dil)][f][dt * C + c]
__global__ void __launch_bounds__(256)
time_stack_nhwc_bwd_kernel(const __nv_bfloat16 *__restrict__ g, float *__restrict__ gx, int C, int T, int F, int Fp,
                           int Cp, int kt, int pt, int dil, long total, int vec) {
  if (vec) {           // one thread = 8 channels: kt 16-byte loads, two 16-byte stores
    const int cvn = C >> 3;
    for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
      const int cv = (int)(i % cvn);
      const long r = i / cvn;
      const int f = (int)(r % F);
      const long bt = r / F;
      const int tp = (int)(bt % T);
      const long b = bt / T;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      for (int dt = 0; dt < kt; ++dt) {
        const int t = tp + pt - dt * dil;
        if (t < 0 || t >= T) continue;
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(g + ((b * T + t) * Fp + f) * Cp + dt * C + cv * 8));
        const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&q);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 w = __bfloat1622float2(h[j]);
          acc[2 * j] += w.x;
          acc[2 * j + 1] += w.y;
        }
      }
      float4 *dst = reinterpret_cast<float4 *>(gx + i * 8);
      dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    return;
  }
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int c = (int)(i % C);
    const long r = i / C;
    const int f = (int)(r % F);
    const long bt = r / F;
    const int tp = (int)(bt % T);
    const long b = bt / T;
    float acc = 0.f;
    for (int dt = 0; dt < kt; ++dt) {
      const int t = tp + pt - dt * dil;
      if (t >= 0 && t < T) acc += __bfloat162float(g[((b * T + t) * Fp + f) * Cp + dt * C + c]);
    }
    gx[i] = acc;
  }
}

}  // namespace rave

extern "C" int rave_time_stack_cl(const float *x, void *out_bf16, int B, int C, int T, int F, int Fp, int Cp, int kt,
                                  int pt, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && out_bf16 && B > 0 && C > 0 && T > 0 && F > 0 && Fp >= F && kt >= 1 && Cp >= kt * C &&
                     Cp <= TS_CP_MAX && Cp % 8 == 0 && C <= TS_CP_MAX / 2 && B <= 65535 && T <= 65535 &&
                     ((uintptr_t)out_bf16 & 15) == 0, "time_stack_cl: bad shape");
  time_stack_cl_kernel<<<dim3(ceil_div(Fp, 32), T, B), 256, 0, (cudaStream_t)stream>>>(
      x, (__nv_bfloat16 *)out_bf16, C, T, F, Fp, Cp, kt, pt);
  RAVE_CHECK_LAUNCH("time_stack_cl");
  return 0;
}

extern "C" int rave_time_stack_cl_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt,
                                      int pt, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(g_bf16 && gx && B > 0 && C > 0 && T > 0 && F > 0 && Fp >= F && kt >= 1 && Cp >= kt * C &&
                     Cp <= TS_CP_MAX && Cp % 8 == 0 && C <= TS_CP_MAX / 2 && B <= 65535 && T <= 65535 &&
                     ((uintptr_t)g_bf16 & 15) == 0, "time_stack_cl_bwd: bad shape");
  time_stack_cl_bwd_kernel<<<dim3(ceil_div(Fp, 32), T, B), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)g_bf16, gx, C, T, F, Fp, Cp, kt, pt);
  RAVE_CHECK_LAUNCH("time_stack_cl_bwd");
  return 0;
}

namespace rave {

static int time_stack_nhwc_launch(const float *x, void *out_bf16, int B, int C, int T, int F, long sb, long st, int Fp,
                                  int Cp, int kt, int pt, int dil, cudaStream_t stream) {
  RAVE_CHECK_ARG(x && out_bf16 && B > 0 && C > 0 && T > 0 && F > 0 && Fp >= F && kt >= 1 && Cp >= kt * C &&
                     Cp % 8 == 0 && dil >= 1 && ((uintptr_t)out_bf16 & 15) == 0, "time_stack_nhwc: bad shape");
  const int vec = (C % 8 == 0) && ((uintptr_t)x & 15) == 0 && sb % 4 == 0 && st % 4 == 0;
  const long total = (long)B * T * Fp * (Cp / 8);
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  time_stack_nhwc_kernel<<<(int)blocks, 256, 0, stream>>>(x, (__nv_bfloat16 *)out_bf16, sb, st, C, T, F, Fp, Cp, kt, pt,
                                                         dil, total, vec);
  RAVE_CHECK_LAUNCH("time_stack_nhwc");
  return 0;
}

static int time_stack_nhwc_bwd_launch(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt,
                                      int pt, int dil, cudaStream_t stream) {
  RAVE_CHECK_ARG(g_bf16 && gx && B > 0 && C > 0 && T > 0 && F > 0 && Fp >= F && kt >= 1 && Cp >= kt * C &&
                     Cp % 8 == 0 && dil >= 1 && ((uintptr_t)g_bf16 & 15) == 0, "time_stack_nhwc_bwd: bad shape");
  const int vec = (C % 8 == 0) && ((uintptr_t)gx & 15) == 0;
  const long total = vec ? (long)B * T * F * (C / 8) : (long)B * T * F * C;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  time_stack_nhwc_bwd_kernel<<<(int)blocks, 256, 0, stream>>>((const __nv_bfloat16 *)g_bf16, gx, C, T, F, Fp, Cp, kt, pt,
                                                             dil, total, vec);
  RAVE_CHECK_LAUNCH("time_stack_nhwc_bwd");
  return 0;
}

}  // namespace rave

extern "C" int rave_time_stack_nhwc(const float *x, void *out_bf16, int B, int C, int T, int F, long sb, long st, int Fp,
                                    int Cp, int kt, int pt, void *stream) {
  return rave::time_stack_nhwc_launch(x, out_bf16, B, C, T, F, sb, st, Fp, Cp, kt, pt, 1, (cudaStream_t)stream);
}

extern "C" int rave_time_stack_nhwc_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt,
                                        int pt, void *stream) {
  return rave::time_stack_nhwc_bwd_launch(g_bf16, gx, B, C, T, F, Fp, Cp, kt, pt, 1, (cudaStream_t)stream);
}

extern "C" int rave_time_stack_nhwc_dil(const float *x, void *out_bf16, int B, int C, int T, int F, long sb, long st,
                                        int Fp, int Cp, int kt, int pt, int dil, void *stream) {
  return rave::time_stack_nhwc_launch(x, out_bf16, B, C, T, F, sb, st, Fp, Cp, kt, pt, dil, (cudaStream_t)stream);
}

extern "C" int rave_time_stack_nhwc_dil_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp,
                                            int kt, int pt, int dil, void *stream) {
  return rave::time_stack_nhwc_bwd_launch(g_bf16, gx, B, C, T, F, Fp, Cp, kt, pt, dil, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// Post-activation feature tap of the Descript discriminator (rave/descript_discriminator.py:59-61, 172-176 + the L1
// feature matching of rave/model.py:353-361 on it): x = chain output holding [real; fake] halves (contiguous, H elements
// each, identical zero padding).  ONE pass: a = LeakyReLU(x) (the feature, and the next layer's input) and
// stats += (sum |a_r - a_f|, sum |a_r|); ONE backward pass:
//   gx_r = (g_r + d0 sgn(a_r - a_f) + d1 sgn(a_r)) * leaky'(a_r),   gx_f = (g_f - d0 sgn(a_r - a_f)) * leaky'(a_f)
// (g = gradient arriving at the feature from its other consumers, or null; d = gradient of the two sums, or null).
// ---------------------------------------------------------------------------------------------
namespace rave {

__device__ __forceinline__ float lk(float x, float slope) { return x > 0.f ? x : slope * x; }
__device__ __forceinline__ float dlk(float a, float slope) { return a > 0.f ? 1.f : slope; }

__global__ void __launch_bounds__(256)
leaky_fm_fwd_kernel(const float *__restrict__ x, float *__restrict__ a, float *__restrict__ stats, long H, float slope,
                    int vec, const BlockSum bs) {
  __shared__ float red0[8], red1[8];
  float s0 = 0.f, s1 = 0.f;
  const long H4 = vec ? (H >> 2) : 0;
  const float4 *xr4 = reinterpret_cast<const float4 *>(x), *xf4 = reinterpret_cast<const float4 *>(x + H);
  float4 *ar4 = reinterpret_cast<float4 *>(a), *af4 = reinterpret_cast<float4 *>(a + H);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < H4; i += (long)gridDim.x * 256) {
    float4 r = __ldg(xr4 + i), f = __ldg(xf4 + i);
    r.x = lk(r.x, slope); r.y = lk(r.y, slope); r.z = lk(r.z, slope); r.w = lk(r.w, slope);
    f.x = lk(f.x, slope); f.y = lk(f.y, slope); f.z = lk(f.z, slope); f.w = lk(f.w, slope);
    ar4[i] = r;
    af4[i] = f;
    s0 += fabsf(r.x - f.x) + fabsf(r.y - f.y) + fabsf(r.z - f.z) + fabsf(r.w - f.w);
    s1 += fabsf(r.x) + fabsf(r.y) + fabsf(r.z) + fabsf(r.w);
  }
  for (long i = (H4 << 2) + blockIdx.x * 256L + threadIdx.x; i < H; i += (long)gridDim.x * 256) {
    const float r = lk(x[i], slope), f = lk(x[H + i], slope);
    a[i] = r;
    a[H + i] = f;
    s0 += fabsf(r - f);
    s1 += fabsf(r);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red0[wid] = s0; red1[wid] = s1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float u0 = 0.f, u1 = 0.f;
    for (int i = 0; i < 8; ++i) { u0 += red0[i]; u1 += red1[i]; }
    block_sum_put(bs, 0, u0);
    block_sum_put(bs, 1, u1);
  }
  block_sum_finish(bs, stats);
}

// The same tap that ALSO writes the next conv's operand (rave_time_stack_nhwc_dil of its own output, kt = 3, pt = dil):
// x rows are (b, t) pairs [2 Rh][F][C]; xs [2 Rh][Fp][3 C] bf16 with xs[(b, t)][f][dt C + c] = a[b][t + (dt - 1) dil][f][c],
// zero outside the T time steps of a batch entry and in the pad columns f >= F.  The element at time t lands in slot 0 of
// row t + dil, slot 1 of row t and slot 2 of row t - dil; the threads of the first / last dil time steps and of the last
// column write the zeros (dil = 1: the MRD's (3, 9) convs; 2, 4: the dilated EncodecConvNet convs).  Saves the stand-alone time-stack pass (read 4 N, write 6 N bytes per layer, 78 launches per step).
__device__ __forceinline__ uint2 pack_bf16x4(float4 v) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  return make_uint2(*reinterpret_cast<const uint32_t *>(&lo), *reinterpret_cast<const uint32_t *>(&hi));
}

__global__ void __launch_bounds__(256)
leaky_fm_stack_fwd_kernel(const float *__restrict__ x, float *__restrict__ a, float *__restrict__ stats,
                          __nv_bfloat16 *__restrict__ xs, long Rh, int T, int F, int C, int Fp, int dil, float slope,
                          const BlockSum bs) {
  __shared__ float red0[8], red1[8];
  float s0 = 0.f, s1 = 0.f;
  const int C4 = C >> 2;
  const int Cp = 3 * C;
  const long H4 = Rh * F * C4;
  const float4 *xr4 = reinterpret_cast<const float4 *>(x), *xf4 = xr4 + H4;
  float4 *ar4 = reinterpret_cast<float4 *>(a), *af4 = ar4 + H4;
  const uint2 zero2 = make_uint2(0u, 0u);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < H4; i += (long)gridDim.x * 256) {
    const int c4 = (int)(i % C4);
    const long rf = i / C4;
    const int f = (int)(rf % F);
    const long r = rf / F;                           // row (b, t) inside a half
    const int t = (int)(r % T);
    float4 rv = __ldg(xr4 + i), fv = __ldg(xf4 + i);
    rv.x = lk(rv.x, slope); rv.y = lk(rv.y, slope); rv.z = lk(rv.z, slope); rv.w = lk(rv.w, slope);
    fv.x = lk(fv.x, slope); fv.y = lk(fv.y, slope); fv.z = lk(fv.z, slope); fv.w = lk(fv.w, slope);
    ar4[i] = rv;
    af4[i] = fv;
    s0 += fabsf(rv.x - fv.x) + fabsf(rv.y - fv.y) + fabsf(rv.z - fv.z) + fabsf(rv.w - fv.w);
    s1 += fabsf(rv.x) + fabsf(rv.y) + fabsf(rv.z) + fabsf(rv.w);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint2 pk = pack_bf16x4(h ? fv : rv);
      const long row = r + (h ? Rh : 0);
      __nv_bfloat16 *base = xs + ((size_t)row * Fp + f) * Cp + 4 * c4;         // slot 0 of this (row, f)
      const size_t row_stride = (size_t)Fp * Cp * dil;
      *reinterpret_cast<uint2 *>(base + C) = pk;                                    // slot 1 of row t
      if (t + dil < T) *reinterpret_cast<uint2 *>(base + row_stride) = pk;          // slot 0 of row t + dil
      else *reinterpret_cast<uint2 *>(base + 2 * C) = zero2;                        // last steps: slot 2 reads t + dil
      if (t >= dil) *reinterpret_cast<uint2 *>(base - row_stride + 2 * C) = pk;     // slot 2 of row t - dil
      else *reinterpret_cast<uint2 *>(base) = zero2;                                // first steps: slot 0 reads t - dil
      if (f == F - 1) {                                                             // pad columns of this row: zeros
        for (int fp = F; fp < Fp; ++fp) {
          __nv_bfloat16 *pz = base + (size_t)(fp - f) * Cp;
          *reinterpret_cast<uint2 *>(pz) = zero2;
          *reinterpret_cast<uint2 *>(pz + C) = zero2;
          *reinterpret_cast<uint2 *>(pz + 2 * C) = zero2;
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red0[wid] = s0; red1[wid] = s1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float u0 = 0.f, u1 = 0.f;
    for (int i = 0; i < 8; ++i) { u0 += red0[i]; u1 += red1[i]; }
    block_sum_put(bs, 0, u0);
    block_sum_put(bs, 1, u1);
  }
  block_sum_finish(bs, stats);
}

__device__ __forceinline__ void leaky_fm_bwd_one(float ar, float af, float gr, float gf, float d0, float d1, float slope,
                                                 float &or_, float &of_) {
  const float s = d0 * sgnf(ar - af);
  or_ = (gr + s + d1 * sgnf(ar)) * dlk(ar, slope);
  of_ = (gf - s) * dlk(af, slope);
}

__global__ void __launch_bounds__(256)
leaky_fm_bwd_kernel(const float *__restrict__ a, const float *__restrict__ g, const float *__restrict__ d,
                    float *__restrict__ gx, long H, float slope, int vec) {
  const float d0 = d ? d[0] : 0.f, d1 = d ? d[1] : 0.f;
  const long H4 = vec ? (H >> 2) : 0;
  const float4 *ar4 = reinterpret_cast<const float4 *>(a), *af4 = reinterpret_cast<const float4 *>(a + H);
  const float4 *gr4 = reinterpret_cast<const float4 *>(g), *gf4 = reinterpret_cast<const float4 *>(g + H);
  float4 *or4 = reinterpret_cast<float4 *>(gx), *of4 = reinterpret_cast<float4 *>(gx + H);
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < H4; i += (long)gridDim.x * 256) {
    const float4 r = __ldg(ar4 + i), f = __ldg(af4 + i);
    const float4 pr = g ? __ldg(gr4 + i) : z, pf = g ? __ldg(gf4 + i) : z;
    float4 o, q;
    leaky_fm_bwd_one(r.x, f.x, pr.x, pf.x, d0, d1, slope, o.x, q.x);
    leaky_fm_bwd_one(r.y, f.y, pr.y, pf.y, d0, d1, slope, o.y, q.y);
    leaky_fm_bwd_one(r.z, f.z, pr.z, pf.z, d0, d1, slope, o.z, q.z);
    leaky_fm_bwd_one(r.w, f.w, pr.w, pf.w, d0, d1, slope, o.w, q.w);
    or4[i] = o;
    of4[i] = q;
  }
  for (long i = (H4 << 2) + blockIdx.x * 256L + threadIdx.x; i < H; i += (long)gridDim.x * 256) {
    float o, q;
    leaky_fm_bwd_one(a[i], a[H + i], g ? g[i] : 0.f, g ? g[H + i] : 0.f, d0, d1, slope, o, q);
    gx[i] = o;
    gx[H + i] = q;
  }
}

// Backward of leaky_fm_stack_fwd in one pass: the gradient reaching a[(b, t)][f][c] through the stacked operand is
//   gxs[(b, t + dil)][f][c] + gxs[(b, t)][f][C + c] + gxs[(b, t - dil)][f][2 C + c]  (rows inside the batch entry only)
// (the adjoint rave_time_stack_nhwc_dil_bwd computes, same summation order), plus `ga` (gradient arriving at the feature
// itself, or null); the feature-matching terms and LeakyReLU' follow as in leaky_fm_bwd_kernel.
__device__ __forceinline__ float4 bf16x4_to_f32(uint2 p) {
  return make_float4(__uint_as_float(p.x << 16), __uint_as_float(p.x & 0xFFFF0000u), __uint_as_float(p.y << 16),
                     __uint_as_float(p.y & 0xFFFF0000u));
}
__device__ __forceinline__ void add4(float4 &a, const float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

__global__ void __launch_bounds__(256)
leaky_fm_stack_bwd_kernel(const float *__restrict__ a, const __nv_bfloat16 *__restrict__ gxs, const float *__restrict__ ga,
                          const float *__restrict__ d, float *__restrict__ gx, long Rh, int T, int F, int C, int Fp,
                          int dil, float slope) {
  const float d0 = d ? d[0] : 0.f, d1 = d ? d[1] : 0.f;
  const int C4 = C >> 2;
  const int Cp = 3 * C;
  const long H4 = Rh * F * C4;
  const size_t row_stride = (size_t)Fp * Cp * dil;
  const float4 *ar4 = reinterpret_cast<const float4 *>(a), *af4 = ar4 + H4;
  const float4 *gr4 = reinterpret_cast<const float4 *>(ga), *gf4 = gr4 + H4;
  float4 *or4 = reinterpret_cast<float4 *>(gx), *of4 = or4 + H4;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < H4; i += (long)gridDim.x * 256) {
    const int c4 = (int)(i % C4);
    const long rf = i / C4;
    const int f = (int)(rf % F);
    const long r = rf / F;
    const int t = (int)(r % T);
    float4 g2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long row = r + (h ? Rh : 0);
      const __nv_bfloat16 *base = gxs + ((size_t)row * Fp + f) * Cp + 4 * c4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t + dil < T) add4(acc, bf16x4_to_f32(__ldg(reinterpret_cast<const uint2 *>(base + row_stride))));
      add4(acc, bf16x4_to_f32(__ldg(reinterpret_cast<const uint2 *>(base + C))));
      if (t >= dil) add4(acc, bf16x4_to_f32(__ldg(reinterpret_cast<const uint2 *>(base - row_stride + 2 * C))));
      if (ga) add4(acc, __ldg((h ? gf4 : gr4) + i));
      g2[h] = acc;
    }
    const float4 rv = __ldg(ar4 + i), fv = __ldg(af4 + i);
    float4 o, q;
    leaky_fm_bwd_one(rv.x, fv.x, g2[0].x, g2[1].x, d0, d1, slope, o.x, q.x);
    leaky_fm_bwd_one(rv.y, fv.y, g2[0].y, g2[1].y, d0, d1, slope, o.y, q.y);
    leaky_fm_bwd_one(rv.z, fv.z, g2[0].z, g2[1].z, d0, d1, slope, o.z, q.z);
    leaky_fm_bwd_one(rv.w, fv.w, g2[0].w, g2[1].w, d0, d1, slope, o.w, q.w);
    or4[i] = o;
    of4[i] = q;
  }
}

}  // namespace rave

extern "C" int rave_leaky_fm_fwd(const float *x, float *a, float *stats, long H, float slope, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && a && stats && H > 0 && slope > 0.f, "leaky_fm_fwd: bad argument");
  const int vec = (H % 4 == 0) && (((uintptr_t)x | (uintptr_t)a) & 15) == 0;
  long blocks = ((vec ? H / 4 : H) + 255) / 256;
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 2, (cudaStream_t)stream)) return rc;
  leaky_fm_fwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(x, a, stats, H, slope, vec, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("leaky_fm_fwd");
  return 0;
}

namespace rave {

static int leaky_fm_stack_fwd_launch(const float *x, float *a, float *stats, void *xs_bf16, long Rh, int T, int F, int C,
                                     int Fp, int dil, float slope, cudaStream_t stream) {
  RAVE_CHECK_ARG(x && a && stats && xs_bf16 && Rh > 0 && T > 0 && Rh % T == 0 && F > 0 && Fp >= F && C > 0 && C % 4 == 0 &&
                     dil >= 1 && slope > 0.f && (((uintptr_t)x | (uintptr_t)a) & 15) == 0 && ((uintptr_t)xs_bf16 & 7) == 0,
                 "leaky_fm_stack_fwd: bad argument (C %% 4 == 0, rows = whole batch entries of T steps, aligned buffers)");
  long blocks = (Rh * F * (C / 4) + 255) / 256;
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 2, stream)) return rc;
  leaky_fm_stack_fwd_kernel<<<(int)blocks, 256, 0, stream>>>(x, a, stats, (__nv_bfloat16 *)xs_bf16, Rh, T, F, C, Fp, dil,
                                                            slope, bs);
  block_sum_end(bs, stream);
  RAVE_CHECK_LAUNCH("leaky_fm_stack_fwd");
  return 0;
}

static int leaky_fm_stack_bwd_launch(const float *a, const void *gxs_bf16, const float *ga, const float *d, float *gx,
                                     long Rh, int T, int F, int C, int Fp, int dil, float slope, cudaStream_t stream) {
  RAVE_CHECK_ARG(a && gxs_bf16 && gx && Rh > 0 && T > 0 && Rh % T == 0 && F > 0 && Fp >= F && C > 0 && C % 4 == 0 &&
                     dil >= 1 && slope > 0.f && (((uintptr_t)a | (uintptr_t)gx | (uintptr_t)ga) & 15) == 0 &&
                     ((uintptr_t)gxs_bf16 & 7) == 0,
                 "leaky_fm_stack_bwd: bad argument (C %% 4 == 0, rows = whole batch entries of T steps, aligned buffers)");
  long blocks = (Rh * F * (C / 4) + 255) / 256;
  blocks = blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks);
  leaky_fm_stack_bwd_kernel<<<(int)blocks, 256, 0, stream>>>(a, (const __nv_bfloat16 *)gxs_bf16, ga, d, gx, Rh, T, F, C,
                                                            Fp, dil, slope);
  RAVE_CHECK_LAUNCH("leaky_fm_stack_bwd");
  return 0;
}

}  // namespace rave

extern "C" int rave_leaky_fm_stack_fwd(const float *x, float *a, float *stats, void *xs_bf16, long Rh, int T, int F, int C,
                                       int Fp, float slope, void *stream) {
  return rave::leaky_fm_stack_fwd_launch(x, a, stats, xs_bf16, Rh, T, F, C, Fp, 1, slope, (cudaStream_t)stream);
}

extern "C" int rave_leaky_fm_stack_bwd(const float *a, const void *gxs_bf16, const float *ga, const float *d, float *gx,
                                       long Rh, int T, int F, int C, int Fp, float slope, void *stream) {
  return rave::leaky_fm_stack_bwd_launch(a, gxs_bf16, ga, d, gx, Rh, T, F, C, Fp, 1, slope, (cudaStream_t)stream);
}

extern "C" int rave_leaky_fm_stack_dil_fwd(const float *x, float *a, float *stats, void *xs_bf16, long Rh, int T, int F,
                                           int C, int Fp, int dil, float slope, void *stream) {
  return rave::leaky_fm_stack_fwd_launch(x, a, stats, xs_bf16, Rh, T, F, C, Fp, dil, slope, (cudaStream_t)stream);
}

extern "C" int rave_leaky_fm_stack_dil_bwd(const float *a, const void *gxs_bf16, const float *ga, const float *d,
                                           float *gx, long Rh, int T, int F, int C, int Fp, int dil, float slope,
                                           void *stream) {
  return rave::leaky_fm_stack_bwd_launch(a, gxs_bf16, ga, d, gx, Rh, T, F, C, Fp, dil, slope, (cudaStream_t)stream);
}

extern "C" int rave_leaky_fm_bwd(const float *a, const float *g, const float *d, float *gx, long H, float slope,
                                 void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(a && gx && (g || d) && H > 0 && slope > 0.f, "leaky_fm_bwd: bad argument");
  const int vec = (H % 4 == 0) && (((uintptr_t)a | (uintptr_t)gx | (uintptr_t)g) & 15) == 0;
  long blocks = ((vec ? H / 4 : H) + 255) / 256;
  blocks = blocks < 1 ? 1 : (blocks > 132 * 16 ? 132 * 16 : blocks);
  leaky_fm_bwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a, g, d, gx, H, slope, vec);
  RAVE_CHECK_LAUNCH("leaky_fm_bwd");
  return 0;
}
