// AdaptiveInstanceNormalization (rave/blocks.py:863-926) in eval mode on the engine's channel-last bf16 streams
// [B][pitch][C] of the v3 chains: the pre-Snake stream h of a Residual(DilatedUnit) is learned from (running mean / std
// of each (b, c) over time) and / or mapped from source to target statistics, between the producing wgmma conv and the
// unit's first conv.  Two launches per layer:
//   adain_cl_stats_kernel : statistics of the L valid rows, the running update of the module's own buffers (every flag
//                           and counter read on the device: one launch sequence serves every style state and can be
//                           captured in a CUDA graph), and the per-(b, c) affine h' = h scale + shift of the transfer;
//   adain_snake_cl_kernel : h' written in place (it is the unit's skip stream) and Snake(h') as the conv operand.
// The sums are fp32 in a fixed order (per thread, then the 32 row lanes, then the row blocks in block order), so two
// runs give the same bits.
#include "common.cuh"

namespace rave {

constexpr int kAdainCh = 64;          // channels per CTA: 8 lanes of 8-channel (16-byte) vectors
constexpr int kAdainRowLanes = 32;

// grid (B * ceil(C / 64), row blocks); block = 8 channel vectors x 32 row lanes.  Partials per CTA: 64 shifted sums
// S1 = sum (x - x0) and 64 sums S2 = sum (x - x0)^2, x0 = row 0 of the same (b, c) (the shift keeps S2 - S1^2 / L
// from cancelling when |mean| >> std).  The last CTA to arrive sums the partials of each (b, c) in block order and
// finalises; it alone reads the counters before it increments one, so no (b, c) sees a counter already advanced.
__global__ void __launch_bounds__(256)
adain_cl_stats_kernel(const __nv_bfloat16 *__restrict__ h, int B, int L, int pitch, int C, float *mean_x, float *std_x,
                      float *mean_y, float *std_y, const float *learn_x, const float *learn_y, float *num_x,
                      float *num_y, float *scale, float *shift, int rows_per_block, const BlockSum bs) {
  __shared__ float red[2][kAdainRowLanes][kAdainCh + 1];
  const bool ly = *learn_y != 0.f, lx = *learn_x != 0.f;
  const bool learn = ly || lx;
  const int cg = (C + kAdainCh - 1) / kAdainCh;
  if (learn) {
    const int b = blockIdx.x / cg, cvl = threadIdx.x & 7, rl = threadIdx.x >> 3;
    const int c0 = (blockIdx.x % cg) * kAdainCh + cvl * 8;
    float s1[8], s2[8], x0[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s1[j] = s2[j] = x0[j] = 0.f;
    if (c0 < C) {
      const __nv_bfloat16 *hb = h + (size_t)b * pitch * C + c0;
      const uint4 q0 = *reinterpret_cast<const uint4 *>(hb);
      const uint32_t w0[4] = {q0.x, q0.y, q0.z, q0.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        x0[2 * j] = __uint_as_float(w0[j] << 16);
        x0[2 * j + 1] = __uint_as_float(w0[j] & 0xFFFF0000u);
      }
      const int r0 = blockIdx.y * rows_per_block, r1 = min(L, r0 + rows_per_block);
      for (int r = r0 + rl; r < r1; r += kAdainRowLanes) {
        const uint4 q = *reinterpret_cast<const uint4 *>(hb + (size_t)r * C);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float d0 = __uint_as_float(w[j] << 16) - x0[2 * j];
          const float d1 = __uint_as_float(w[j] & 0xFFFF0000u) - x0[2 * j + 1];
          s1[2 * j] += d0;
          s2[2 * j] = fmaf(d0, d0, s2[2 * j]);
          s1[2 * j + 1] += d1;
          s2[2 * j + 1] = fmaf(d1, d1, s2[2 * j + 1]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      red[0][rl][cvl * 8 + j] = s1[j];
      red[1][rl][cvl * 8 + j] = s2[j];
    }
    __syncthreads();
    if (threadIdx.x < 2 * kAdainCh) {
      const int k = threadIdx.x / kAdainCh, i = threadIdx.x % kAdainCh;
      float t = 0.f;
#pragma unroll 8
      for (int r = 0; r < kAdainRowLanes; ++r) t += red[k][r][i];
      block_sum_put(bs, threadIdx.x, t);
    }
    // limit 0: block_sum_finish only serves as the arrival ticket; the last CTA reduces the partials itself (below)
    if (!block_sum_finish(bs, nullptr)) return;
  } else if (blockIdx.x != 0 || blockIdx.y != 0) {
    return;                      // nothing to learn: the first CTA computes the affine from the buffers alone
  }
  // ---- last CTA (or the only one working): finalise every (b, c)
  const float ny = *num_y, nx = *num_x;
  const bool apply = !ly && (lx ? nx + 1.f : nx) != 0.f && ny != 0.f;
  const unsigned gx = gridDim.x, per = gridDim.y;
  for (int o = threadIdx.x; o < B * C; o += blockDim.x) {
    const int b = o / C, c = o % C;
    if (learn) {
      const unsigned g = (unsigned)(b * cg + c / kAdainCh), i = c % kAdainCh;
      float t1 = 0.f, t2 = 0.f;
      for (unsigned j = 0; j < per; ++j) {
        const float *p = bs.part + (size_t)(g + gx * j) * (2 * kAdainCh);
        t1 += __ldcg(p + i);
        t2 += __ldcg(p + kAdainCh + i);
      }
      const float xs = __bfloat162float(h[(size_t)b * pitch * C + c]);
      const float n = (float)L;
      // torch.std: unbiased (N - 1); L = 1 gives 0 / 0 = NaN, as the reference does
      const float var = fmaxf(t2 - t1 * (t1 / n), 0.f) / (n - 1.f);
      const float mean = xs + t1 / n, sd = sqrtf(var);
      float *m = ly ? mean_y : mean_x, *s = ly ? std_y : std_x;
      const float k = (ly ? ny : nx) + 1.f;
      m[o] += (mean - m[o]) / k;
      s[o] += (sd - s[o]) / k;
    }
    float sc = 1.f, sh = 0.f;
    if (apply) {
      sc = std_y[o] / (std_x[o] + 1e-5f);
      sh = mean_y[o] - mean_x[o] * sc;
    }
    scale[o] = sc;
    shift[o] = sh;
  }
  __syncthreads();               // every (b, c) has read the counters
  if (threadIdx.x == 0) {
    if (ly)
      *num_y = ny + 1.f;
    else if (lx)
      *num_x = nx + 1.f;
  }
}

// h' = h scale[b, c] + shift[b, c] on rows < L, written back into h (skipped where the affine is the identity) and
// a = Snake(h') as the next conv's operand; slack rows of a are zero (those of h stay as they are: zero).  With scale
// 1, shift 0 the operand is bit for bit what snake_cl_fwd_kernel writes.
__global__ void __launch_bounds__(256)
adain_snake_cl_kernel(__nv_bfloat16 *__restrict__ h, const float *__restrict__ alpha, const float *__restrict__ scale,
                      const float *__restrict__ shift, __nv_bfloat16 *__restrict__ a, long n_vec, int cv, int L,
                      int pitch) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n_vec; i += (long)gridDim.x * 256) {
    const long row = i / cv;
    const int c0 = (int)(i % cv) * 8, l = (int)(row % pitch);
    if (l >= L) {
      *reinterpret_cast<uint4 *>(a + i * 8) = make_uint4(0, 0, 0, 0);
      continue;
    }
    const size_t bc = (size_t)(row / pitch) * cv * 8 + c0;
    const uint4 q = *reinterpret_cast<const uint4 *>(h + i * 8);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t o[4], hn[4];
    bool ident = true;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sc0 = __ldg(scale + bc + 2 * j), sc1 = __ldg(scale + bc + 2 * j + 1);
      const float sh0 = __ldg(shift + bc + 2 * j), sh1 = __ldg(shift + bc + 2 * j + 1);
      ident = ident && sc0 == 1.f && sc1 == 1.f && sh0 == 0.f && sh1 == 0.f;
      const __nv_bfloat162 hh = __floats2bfloat162_rn(fmaf(__uint_as_float(w[j] << 16), sc0, sh0),
                                                      fmaf(__uint_as_float(w[j] & 0xFFFF0000u), sc1, sh1));
      hn[j] = *reinterpret_cast<const uint32_t *>(&hh);
      const float x0 = __uint_as_float(hn[j] << 16), x1 = __uint_as_float(hn[j] & 0xFFFF0000u);
      const float a0 = __ldg(alpha + c0 + 2 * j), a1 = __ldg(alpha + c0 + 2 * j + 1);
      const float s0 = sinf(a0 * x0), s1 = sinf(a1 * x1);
      const __nv_bfloat162 r = __floats2bfloat162_rn(x0 + s0 * s0 / (a0 + 1e-9f), x1 + s1 * s1 / (a1 + 1e-9f));
      o[j] = *reinterpret_cast<const uint32_t *>(&r);
    }
    if (!ident) *reinterpret_cast<uint4 *>(h + i * 8) = make_uint4(hn[0], hn[1], hn[2], hn[3]);
    *reinterpret_cast<uint4 *>(a + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace rave

extern "C" int rave_adain_cl_stats(const void *h_bf16, int B, int L, int pitch, int C, float *mean_x, float *std_x,
                                   float *mean_y, float *std_y, const float *learn_x, const float *learn_y,
                                   float *num_update_x, float *num_update_y, int max_batch, float *scale, float *shift,
                                   void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h_bf16 && mean_x && std_x && mean_y && std_y && learn_x && learn_y && num_update_x && num_update_y &&
                     scale && shift,
                 "adain_cl_stats: null argument");
  RAVE_CHECK_ARG(B > 0 && B <= max_batch, "adain_cl_stats: batch %d exceeds the %d rows of the statistics buffers", B,
                 max_batch);
  RAVE_CHECK_ARG(C > 0 && C % 8 == 0 && L > 0 && pitch >= L && ((uintptr_t)h_bf16 & 15) == 0,
                 "adain_cl_stats: bad argument (C %d %% 8, L %d <= pitch %d, 16-byte rows)", C, L, pitch);
  const int cg = (C + kAdainCh - 1) / kAdainCh;
  const long gx = (long)cg * B;
  long gy = (L + 255) / 256;                    // >= 256 rows per CTA, about two waves of CTAs in all
  const long cap = (132L * 2 + gx - 1) / gx;
  if (gy > cap) gy = cap;
  if (gy < 1) gy = 1;
  const int rpb = (int)((L + gy - 1) / gy);
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, gx * gy, 2 * kAdainCh, (cudaStream_t)stream)) return rc;
  bs.limit = 0;
  adain_cl_stats_kernel<<<dim3((unsigned)gx, (unsigned)gy), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)h_bf16, B, L, pitch, C, mean_x, std_x, mean_y, std_y, learn_x, learn_y, num_update_x,
      num_update_y, scale, shift, rpb, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("adain_cl_stats");
  return 0;
}

extern "C" int rave_adain_snake_cl_fwd(void *h_bf16, const float *alpha, const float *scale, const float *shift,
                                       void *a_bf16, int B, int L, int pitch, int C, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h_bf16 && alpha && scale && shift && a_bf16, "adain_snake_cl_fwd: null argument");
  RAVE_CHECK_ARG(B > 0 && C > 0 && C % 8 == 0 && L > 0 && pitch >= L &&
                     (((uintptr_t)h_bf16 | (uintptr_t)a_bf16) & 15) == 0,
                 "adain_snake_cl_fwd: bad argument (C %d %% 8, L %d <= pitch %d, 16-byte rows)", C, L, pitch);
  const long n_vec = (long)B * pitch * (C / 8);
  long blocks = (n_vec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  adain_snake_cl_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16 *)h_bf16, alpha, scale, shift, (__nv_bfloat16 *)a_bf16, n_vec, C / 8, L, pitch);
  RAVE_CHECK_LAUNCH("adain_snake_cl_fwd");
  return 0;
}
