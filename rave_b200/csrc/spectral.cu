// Fused multi-scale spectral distance (SURVEY row 8f.1): the elementwise / reduction tail of
// core.AudioDistanceV1 (rave/core.py:322-344) + mean_difference (236-252) applied to the complex STFTs of
// the input (X) and of the reconstruction (Y), one scale per launch:
//     lin = mean((|X|-|Y|)^2) / mean(|X|^2)          log = mean(| log(|X|+eps) - log(|Y|+eps) |)
// forward : stats[0] += sum (|X|-|Y|)^2, stats[1] += sum |X|^2, stats[2] += sum |log(|X|+eps) - log(|Y|+eps)|;
//           the last block to finish (block-order sums, see BlockSum) writes the distance stats[4] = s0/s1 + s2/n, so the
//           scalar tail costs no extra launches
// backward: dY = ( c_lin * -2 (|X|-|Y|) + c_log * -sgn(logX - logY) / (|Y|+eps) ) * Y/|Y|, c_lin = g/s1, c_log = g/n
//           with the upstream gradient g read from device memory
//           (PyTorch's convention for the gradient of a real loss w.r.t. a complex tensor through abs()).
// Replaces ~14 ATen elementwise/reduce kernels per scale forward and ~25 backward with one kernel each.
#include "common.cuh"

namespace rave {

__global__ void __launch_bounds__(256)
spectral_stats_kernel(const float2 *__restrict__ X, const float2 *__restrict__ Y, float *__restrict__ stats, long n,
                      float eps, const BlockSum bs) {
  __shared__ float red[3][8];
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float2 x = X[i], y = Y[i];
    const float ax = sqrtf(x.x * x.x + x.y * x.y);
    const float ay = sqrtf(y.x * y.x + y.y * y.y);
    const float d = ax - ay;
    s0 = fmaf(d, d, s0);
    s1 = fmaf(ax, ax, s1);
    s2 += fabsf(logf(ax + eps) - logf(ay + eps));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[0][wid] = s0; red[1][wid] = s1; red[2][wid] = s2; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
    block_sum_put(bs, threadIdx.x, t);
  }
  if (block_sum_finish(bs, stats) && threadIdx.x == 0) stats[4] = stats[0] / stats[1] + stats[2] / (float)n;
}

__global__ void __launch_bounds__(256)
spectral_grad_kernel(const float2 *__restrict__ X, const float2 *__restrict__ Y, float2 *__restrict__ dY,
                     const float *__restrict__ stats, const float *__restrict__ gup, long n, float eps) {
  const float g = gup[0];
  const float c_lin = g / stats[1], c_log = g / (float)n;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float2 x = X[i], y = Y[i];
    const float ax = sqrtf(x.x * x.x + x.y * x.y);
    const float ay = sqrtf(y.x * y.x + y.y * y.y);
    const float dl = logf(ax + eps) - logf(ay + eps);
    const float sg = dl > 0.f ? 1.f : (dl < 0.f ? -1.f : 0.f);
    const float dmag = c_lin * (-2.f) * (ax - ay) - c_log * sg / (ay + eps);
    const float inv = ay > 0.f ? dmag / ay : 0.f;
    dY[i] = make_float2(y.x * inv, y.y * inv);
  }
}

// ---------------------------------------------------------------------------------------------
// STFT framing (torch.stft(center=True, pad_mode="reflect") minus the FFT itself, rave/core.py:286-306):
//   frames[n][f][t] = w[t] * x[n][reflect(f*hop + t - n_fft/2)]          reflect(i) = -i (i<0), 2(T-1)-i (i>=T)
// one kernel instead of reflection_pad1d + as_strided + mul, and one kernel for the adjoint (window, overlap-add,
// fold of the reflected borders) instead of mul + index_add + reflection_pad1d_backward.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
stft_frames_kernel(const float *__restrict__ x, const float *__restrict__ w, float *__restrict__ frames, long total4,
                   int T, int n_fft, int hop, int F, int vec_ok) {
  // one thread = 4 consecutive samples of one frame (n_fft is a power of two >= 16: shifts, one division by F)
  const int h = n_fft >> 1;
  const int q = n_fft >> 2;                   // float4 per frame
  const int qs = 31 - __clz(q);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total4; i += (long)gridDim.x * 256) {
    const int t = (int)(i & (q - 1)) << 2;
    const long nf = i >> qs;
    const int f = (int)(nf % F);
    const long n = nf / F;
    const int j0 = f * hop + t - h;
    const float4 ww = __ldg(reinterpret_cast<const float4 *>(w + t));
    const float *xn = x + n * T;
    float4 xv;
    if (vec_ok && j0 >= 0 && j0 + 3 < T) {
      xv = __ldg(reinterpret_cast<const float4 *>(xn + j0));
    } else {
      float e[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        int j = j0 + u;
        if (j < 0) j = -j;
        if (j >= T) j = 2 * (T - 1) - j;
        e[u] = __ldg(xn + j);
      }
      xv = make_float4(e[0], e[1], e[2], e[3]);
    }
    reinterpret_cast<float4 *>(frames)[i] = make_float4(ww.x * xv.x, ww.y * xv.y, ww.z * xv.z, ww.w * xv.w);
  }
}

__device__ __forceinline__ float stft_ola_at(const float *__restrict__ d, const float *__restrict__ w, int p, int n_fft,
                                             int hop, int F) {
  // sum over the frames that cover padded position p
  float acc = 0.f;
  int f_hi = p / hop;
  if (f_hi > F - 1) f_hi = F - 1;
  int f_lo = (p - n_fft + hop) / hop;          // ceil((p - n_fft + 1) / hop) for p - n_fft + 1 >= 0
  if (p - n_fft + 1 <= 0) f_lo = 0;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int t = p - f * hop;
    acc = fmaf(__ldg(w + t), __ldg(d + (size_t)f * n_fft + t), acc);
  }
  return acc;
}

__global__ void __launch_bounds__(256)
stft_frames_bwd_kernel(const float *__restrict__ dframes, const float *__restrict__ w, float *__restrict__ dx, long total,
                       int T, int n_fft, int hop, int F) {
  const int h = n_fft >> 1;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int j = (int)(i % T);
    const long n = i / T;
    const float *d = dframes + (size_t)n * F * n_fft;
    float acc = stft_ola_at(d, w, j + h, n_fft, hop, F);
    if (j >= 1 && j <= h) acc += stft_ola_at(d, w, h - j, n_fft, hop, F);
    if (j <= T - 2 && j >= T - 1 - h) acc += stft_ola_at(d, w, 2 * (T - 1) - j + h, n_fft, hop, F);
    dx[i] = acc;
  }
}

// Uncentred framing (torchaudio Spectrogram(center=False, normalized=True) of the multi-scale spectral discriminator,
// rave/discriminator.py:12-20), F = 1 + (T - n_fft) / hop frames, no padding:
//   frames[n][f][t] = s * w[t] * x[n][f*hop + t]           s = 1 / ||w||_2 for normalized=True
// adjoint: dx[n][j] = s * sum over the frames f covering j of w[j - f*hop] * dframes[n][f][j - f*hop] (a gather: one
// thread per output sample, no atomics); samples past the last frame get zero.
__global__ void __launch_bounds__(256)
stft_frames_valid_kernel(const float *__restrict__ x, const float *__restrict__ w, float *__restrict__ frames, long total4,
                         int T, int n_fft, int hop, int F, float s, int vec_ok) {
  const int q = n_fft >> 2;                   // float4 per frame
  const int qs = 31 - __clz(q);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total4; i += (long)gridDim.x * 256) {
    const int t = (int)(i & (q - 1)) << 2;
    const long nf = i >> qs;
    const int f = (int)(nf % F);
    const long n = nf / F;
    const float *xn = x + n * T + (long)f * hop + t;
    const float4 ww = __ldg(reinterpret_cast<const float4 *>(w + t));
    const float4 xv = vec_ok ? __ldg(reinterpret_cast<const float4 *>(xn))
                             : make_float4(__ldg(xn), __ldg(xn + 1), __ldg(xn + 2), __ldg(xn + 3));
    reinterpret_cast<float4 *>(frames)[i] =
        make_float4(s * ww.x * xv.x, s * ww.y * xv.y, s * ww.z * xv.z, s * ww.w * xv.w);
  }
}

__global__ void __launch_bounds__(256)
stft_frames_valid_bwd_kernel(const float *__restrict__ dframes, const float *__restrict__ w, float *__restrict__ dx,
                             long total, int T, int n_fft, int hop, int F, float s) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int j = (int)(i % T);
    const long n = i / T;
    dx[i] = s * stft_ola_at(dframes + (size_t)n * F * n_fft, w, j, n_fft, hop, F);
  }
}

// Gradient of y = rfft(x) (last axis, length n) as the input of ONE c2r transform: Z[k] = G[k] * n * (k == 0 || k == n/2
// ? 1 : 1/2), imaginary parts of the DC and Nyquist bins dropped (cuFFT's C2R result is unspecified for a non-Hermitian
// input; those parts carry no gradient).  dx = irfft(Z, n).  G: [N][F][bins] complex64 with arbitrary strides.
__global__ void __launch_bounds__(256)
rfft_bwd_scale_kernel(const float2 *__restrict__ G, float2 *__restrict__ Z, long total, int F, int bins, long sN, long sF,
                      long sB, float n) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int k = (int)(i % bins);
    const long nf = i / bins;
    const int f = (int)(nf % F);
    const long b = nf / F;
    const float2 g = G[b * sN + f * sF + k * sB];
    const bool edge = (k == 0) || (k == bins - 1);
    const float sc = edge ? n : 0.5f * n;
    Z[i] = make_float2(g.x * sc, edge ? 0.f : g.y * sc);
  }
}

}  // namespace rave

extern "C" int rave_rfft_bwd_scale(const void *G_c64, void *Z_c64, long N, int F, int bins, long sN, long sF, long sB,
                                   void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(G_c64 && Z_c64 && N > 0 && F > 0 && bins > 1, "rfft_bwd_scale: bad argument");
  const long total = N * F * bins;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  rfft_bwd_scale_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const float2 *)G_c64, (float2 *)Z_c64, total, F,
                                                                       bins, sN, sF, sB, (float)(2 * (bins - 1)));
  RAVE_CHECK_LAUNCH("rfft_bwd_scale");
  return 0;
}

extern "C" int rave_stft_frames(const float *x, const float *window, float *frames, int N, int T, int n_fft, int hop,
                                void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && window && frames && N > 0 && T > n_fft / 2 && n_fft >= 16 && (n_fft & (n_fft - 1)) == 0 &&
                     hop > 0 && n_fft % hop == 0 && hop % 4 == 0,
                 "stft_frames: bad argument (reflect padding needs T > n_fft/2; n_fft a power of two >= 16, 4 | hop | n_fft)");
  const int F = 1 + T / hop;
  const long total4 = (long)N * F * (n_fft / 4);
  long blocks = (total4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  const int vec_ok = (T % 4 == 0) && (((uintptr_t)x & 15) == 0);
  stft_frames_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(x, window, frames, total4, T, n_fft, hop, F, vec_ok);
  RAVE_CHECK_LAUNCH("stft_frames");
  return 0;
}

extern "C" int rave_stft_frames_bwd(const float *dframes, const float *window, float *dx, int N, int T, int n_fft,
                                    int hop, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dframes && window && dx && N > 0 && T > n_fft / 2 && n_fft >= 2 && hop > 0 && n_fft % hop == 0,
                 "stft_frames_bwd: bad argument");
  const int F = 1 + T / hop;
  const long total = (long)N * T;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  stft_frames_bwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(dframes, window, dx, total, T, n_fft, hop, F);
  RAVE_CHECK_LAUNCH("stft_frames_bwd");
  return 0;
}

extern "C" int rave_stft_frames_valid(const float *x, const float *window, float *frames, int N, int T, int n_fft, int hop,
                                      float scale, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && window && frames && N > 0 && T >= n_fft && n_fft >= 16 && (n_fft & (n_fft - 1)) == 0 && hop > 0,
                 "stft_frames_valid: bad argument (T >= n_fft, n_fft a power of two >= 16)");
  const int F = 1 + (T - n_fft) / hop;
  const long total4 = (long)N * F * (n_fft / 4);
  long blocks = (total4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  const int vec_ok = (T % 4 == 0) && (hop % 4 == 0) && (((uintptr_t)x & 15) == 0);
  stft_frames_valid_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(x, window, frames, total4, T, n_fft, hop, F,
                                                                          scale, vec_ok);
  RAVE_CHECK_LAUNCH("stft_frames_valid");
  return 0;
}

extern "C" int rave_stft_frames_valid_bwd(const float *dframes, const float *window, float *dx, int N, int T, int n_fft,
                                          int hop, float scale, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dframes && window && dx && N > 0 && T >= n_fft && n_fft >= 16 && hop > 0,
                 "stft_frames_valid_bwd: bad argument");
  const int F = 1 + (T - n_fft) / hop;
  const long total = (long)N * T;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  stft_frames_valid_bwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(dframes, window, dx, total, T, n_fft, hop,
                                                                              F, scale);
  RAVE_CHECK_LAUNCH("stft_frames_valid_bwd");
  return 0;
}

extern "C" int rave_spectral_stats(const void *X, const void *Y, float *stats, long n, float eps, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(X && Y && stats && n > 0, "spectral_stats: bad argument");
  long blocks = (n + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 3, (cudaStream_t)stream)) return rc;
  spectral_stats_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const float2 *)X, (const float2 *)Y, stats, n,
                                                                       eps, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("spectral_stats");
  return 0;
}

extern "C" int rave_spectral_grad(const void *X, const void *Y, void *dY, const float *stats, const float *gup, long n,
                                  float eps, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(X && Y && dY && stats && gup && n > 0, "spectral_grad: bad argument");
  long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  spectral_grad_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const float2 *)X, (const float2 *)Y,
                                                                      (float2 *)dY, stats, gup, n, eps);
  RAVE_CHECK_LAUNCH("spectral_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Mel front end of the hybrid encoder (rave/model.py:238-242 with torchaudio.transforms.MelSpectrogram(normalized=True),
// configs/hybrid.gin): from the complex STFT X[n][f][k] (n = b*C + c, centred frames, cuFFT),
//     out[b][c*M + m][f] = log1p( scale * sum_{k in [lo_m, hi_m)} fb_m[k - lo_m] |X[n][f][k]|^2 ),   f < F - 1
// scale = 1 / sum(w^2).  The HTK filter bank is banded (each band spans a contiguous bin range), so the host passes
// per-band [lo, hi) and the packed nonzero weights.  One CTA = one signal n and MEL_FT frames: |X|^2 of those frames
// goes through shared memory, one thread per (band, frame) output.
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int MEL_FT = 8;

__global__ void __launch_bounds__(256)
mel_log1p_kernel(const float2 *__restrict__ X, const int *__restrict__ band, const float *__restrict__ wts,
                 float *__restrict__ out, int F, int bins, int M, int nnz, float scale) {
  extern __shared__ float sm[];
  float *P = sm;                          // [MEL_FT][bins]
  float *W = P + MEL_FT * bins;           // [nnz]
  int *bd = reinterpret_cast<int *>(W + nnz);   // [M][3]: lo, hi, offset into W
  const int n = blockIdx.y, f0 = blockIdx.x * MEL_FT;
  const int Fo = F - 1;                   // the last frame is dropped
  const int nf = min(MEL_FT, Fo - f0);
  const float2 *Xn = X + ((size_t)n * F + f0) * bins;
  for (int i = threadIdx.x; i < nf * bins; i += blockDim.x) {
    const float2 v = Xn[i];
    P[i] = fmaf(v.x, v.x, v.y * v.y);
  }
  for (int i = threadIdx.x; i < nnz; i += blockDim.x) W[i] = wts[i];
  for (int i = threadIdx.x; i < 3 * M; i += blockDim.x) bd[i] = band[i];
  __syncthreads();
  for (int o = threadIdx.x; o < M * MEL_FT; o += blockDim.x) {
    const int m = o / MEL_FT, f = o % MEL_FT;
    if (f >= nf) continue;
    const int lo = bd[3 * m], hi = bd[3 * m + 1], off = bd[3 * m + 2];
    const float *p = P + f * bins;
    float acc = 0.f;
    for (int k = lo; k < hi; ++k) acc = fmaf(W[off + k - lo], p[k], acc);
    out[((size_t)n * M + m) * Fo + f0 + f] = log1pf(scale * acc);
  }
}

// Gradient of mel_log1p_kernel with respect to X (the receptive-field probe of a mel-input model differentiates through
// the front end):  dX[n][f][k] = 2 scale X[n][f][k] sum_m w_m[k] dy[n][m][f] / (1 + mel[n][m][f]), zero for the dropped
// last frame.  Same tiling as the forward: the band sums are recomputed from |X|^2 in shared memory, then one thread per
// (frame, bin) adds the bands covering bin k in band order.
__global__ void __launch_bounds__(256)
mel_log1p_bwd_kernel(const float2 *__restrict__ X, const int *__restrict__ band, const float *__restrict__ wts,
                     const float *__restrict__ dy, float2 *__restrict__ dX, int F, int bins, int M, int nnz, float scale) {
  extern __shared__ float sm[];
  float *P = sm;                          // [MEL_FT][bins]
  float *W = P + MEL_FT * bins;           // [nnz]
  float *G = W + nnz;                     // [M][MEL_FT]: dy / (1 + mel)
  int *bd = reinterpret_cast<int *>(G + M * MEL_FT);
  const int n = blockIdx.y, f0 = blockIdx.x * MEL_FT;
  const int Fo = F - 1;
  const int nf = min(MEL_FT, F - f0);     // frames of this CTA, the dropped one included
  const int nv = min(MEL_FT, Fo - f0);    // frames with an output
  const float2 *Xn = X + ((size_t)n * F + f0) * bins;
  float2 *dXn = dX + ((size_t)n * F + f0) * bins;
  for (int i = threadIdx.x; i < nf * bins; i += blockDim.x) {
    const float2 v = Xn[i];
    P[i] = fmaf(v.x, v.x, v.y * v.y);
  }
  for (int i = threadIdx.x; i < nnz; i += blockDim.x) W[i] = wts[i];
  for (int i = threadIdx.x; i < 3 * M; i += blockDim.x) bd[i] = band[i];
  __syncthreads();
  for (int o = threadIdx.x; o < M * MEL_FT; o += blockDim.x) {
    const int m = o / MEL_FT, f = o % MEL_FT;
    float g = 0.f;
    if (f < nv) {
      const int lo = bd[3 * m], hi = bd[3 * m + 1], off = bd[3 * m + 2];
      const float *p = P + f * bins;
      float acc = 0.f;
      for (int k = lo; k < hi; ++k) acc = fmaf(W[off + k - lo], p[k], acc);
      g = dy[((size_t)n * M + m) * Fo + f0 + f] / (1.f + scale * acc);
    }
    G[o] = g;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nf * bins; i += blockDim.x) {
    const int f = i / bins, k = i % bins;
    float s = 0.f;
    if (f < nv)
      for (int m = 0; m < M; ++m) {
        const int lo = bd[3 * m], hi = bd[3 * m + 1];
        if (k >= lo && k < hi) s = fmaf(W[bd[3 * m + 2] + k - lo], G[m * MEL_FT + f], s);
      }
    const float2 v = Xn[i];
    const float c = 2.f * scale * s;
    dXn[i] = make_float2(c * v.x, c * v.y);
  }
}

}  // namespace rave

extern "C" int rave_mel_log1p_fwd(const void *X_c64, const int *band, const float *weights, float *out, int N, int F,
                                  int bins, int M, int nnz, float scale, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(X_c64 && band && weights && out && N > 0 && F > 1 && bins > 0 && M > 0 && nnz > 0 && N <= 65535,
                 "mel_log1p_fwd: bad argument");
  const size_t smem = ((size_t)MEL_FT * bins + nnz + 3 * M) * 4;
  RAVE_CHECK_ARG(smem <= 48 * 1024, "mel_log1p_fwd: %d bins / %d filter weights / %d bands need %zu bytes of shared memory "
                 "(at most 48 KB)", bins, nnz, M, smem);
  dim3 grid(ceil_div(F - 1, MEL_FT), N);
  mel_log1p_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>((const float2 *)X_c64, band, weights, out, F, bins, M, nnz,
                                                             scale);
  RAVE_CHECK_LAUNCH("mel_log1p_fwd");
  return 0;
}

extern "C" int rave_mel_log1p_bwd(const void *X_c64, const int *band, const float *weights, const float *dy, void *dX_c64,
                                  int N, int F, int bins, int M, int nnz, float scale, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(X_c64 && band && weights && dy && dX_c64 && N > 0 && F > 1 && bins > 0 && M > 0 && nnz > 0 &&
                 N <= 65535, "mel_log1p_bwd: bad argument");
  const size_t smem = ((size_t)MEL_FT * bins + nnz + (size_t)M * MEL_FT + 3 * M) * 4;
  RAVE_CHECK_ARG(smem <= 48 * 1024, "mel_log1p_bwd: %d bins / %d filter weights / %d bands need %zu bytes of shared memory "
                 "(at most 48 KB)", bins, nnz, M, smem);
  dim3 grid(ceil_div(F, MEL_FT), N);
  mel_log1p_bwd_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>((const float2 *)X_c64, band, weights, dy,
                                                                 (float2 *)dX_c64, F, bins, M, nnz, scale);
  RAVE_CHECK_LAUNCH("mel_log1p_bwd");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// NoiseGeneratorV2 tail (rave/blocks.py:284-292, rave/core.py:20-21,48-81): band amplitudes -> FIR -> filtered
// uniform noise, in ONE kernel.  The reference goes mod_sigmoid -> irfft -> roll -> hann -> pad/crop -> roll
// (amp_to_impulse_response) and then a zero-padded rfft * rfft -> irfft (fft_convolve): 4 FFT launches and ~15
// elementwise kernels for what is, per (batch, frame, channel) group, a [target x bands] LINEAR map of the amplitudes
// (every step of amp_to_impulse_response is linear) followed by a causal convolution of `target` samples:
//     amp[k]   = 2 sigmoid(h[b][c*NB + k][t] - 5)^2.3 + 1e-7
//     ir[n]    = sum_k M[n][k] amp[k]                       (M: the reference pipeline applied to the identity, host)
//     out[b][c][t*TS + i] = sum_{j <= i} noise[b][t][c][j] * ir[i - j]
// h: [B][C*NB][T] conv output (NCL), noise: [B][T][C][TS], out: [B][C][T*TS].  One thread per (b, c, t).
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int NF_MAX_TS = 16;     // target_size (prod of the noise ratios; 8 in configs/v2_small.gin:42-57)
constexpr int NF_MAX_NB = 64;     // noise bands (32)

__device__ __forceinline__ float mod_sigmoid_f(float x) {
  const float s = 1.f / (1.f + __expf(-x));
  return 2.f * powf(s, 2.3f) + 1e-7f;
}

__global__ void __launch_bounds__(128)
noise_fir_fwd_kernel(const float *__restrict__ h, const float *__restrict__ M, const float *__restrict__ noise,
                     float *__restrict__ out, int C, int NB, int T, int TS) {
  extern __shared__ float Ms[];            // [TS][NB]
  for (int i = threadIdx.x; i < TS * NB; i += blockDim.x) Ms[i] = M[i];
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  float ir[NF_MAX_TS];
#pragma unroll
  for (int n = 0; n < NF_MAX_TS; ++n) ir[n] = 0.f;
  const float *hp = h + ((size_t)b * C * NB + (size_t)c * NB) * T + t;
  for (int k = 0; k < NB; ++k) {
    const float a = mod_sigmoid_f(hp[(size_t)k * T] - 5.f);
#pragma unroll
    for (int n = 0; n < NF_MAX_TS; ++n)
      if (n < TS) ir[n] = fmaf(Ms[n * NB + k], a, ir[n]);
  }
  const float *np_ = noise + (((size_t)b * T + t) * C + c) * TS;
  float nz[NF_MAX_TS];
#pragma unroll
  for (int j = 0; j < NF_MAX_TS; ++j) nz[j] = j < TS ? np_[j] : 0.f;
  float *op = out + ((size_t)b * C + c) * T * TS + (size_t)t * TS;
#pragma unroll
  for (int i = 0; i < NF_MAX_TS; ++i) {
    if (i >= TS) break;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < NF_MAX_TS; ++j)
      if (j <= i) acc = fmaf(nz[j], ir[i - j], acc);
    op[i] = acc;
  }
}

// dh[b][c*NB + k][t] = mod_sigmoid'(h - 5) * sum_n M[n][k] * dir[n],   dir[n] = sum_{i >= n} dout[i] noise[i - n]
__global__ void __launch_bounds__(128)
noise_fir_bwd_kernel(const float *__restrict__ h, const float *__restrict__ M, const float *__restrict__ noise,
                     const float *__restrict__ dout, float *__restrict__ dh, int C, int NB, int T, int TS) {
  extern __shared__ float Ms[];
  for (int i = threadIdx.x; i < TS * NB; i += blockDim.x) Ms[i] = M[i];
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  const float *np_ = noise + (((size_t)b * T + t) * C + c) * TS;
  const float *gp = dout + ((size_t)b * C + c) * T * TS + (size_t)t * TS;
  float nz[NF_MAX_TS], go[NF_MAX_TS], dir[NF_MAX_TS];
#pragma unroll
  for (int j = 0; j < NF_MAX_TS; ++j) {
    nz[j] = j < TS ? np_[j] : 0.f;
    go[j] = j < TS ? gp[j] : 0.f;
  }
#pragma unroll
  for (int n = 0; n < NF_MAX_TS; ++n) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < NF_MAX_TS; ++i)
      if (i >= n && i < TS) acc = fmaf(go[i], nz[i - n], acc);
    dir[n] = acc;
  }
  const size_t base = ((size_t)b * C * NB + (size_t)c * NB) * T + t;
  for (int k = 0; k < NB; ++k) {
    float da = 0.f;
#pragma unroll
    for (int n = 0; n < NF_MAX_TS; ++n)
      if (n < TS) da = fmaf(Ms[n * NB + k], dir[n], da);
    // d/dx [2 s^2.3] = 4.6 s^2.3 (1 - s),  s = sigmoid(x)
    const float x = h[base + (size_t)k * T] - 5.f;
    const float s = 1.f / (1.f + __expf(-x));
    dh[base + (size_t)k * T] = da * 4.6f * powf(s, 2.3f) * (1.f - s);
  }
}

}  // namespace rave

extern "C" int rave_noise_fir_fwd(const float *h, const float *M, const float *noise, float *out, int B, int C, int NB,
                                  int T, int TS, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h && M && noise && out && B > 0 && C > 0 && T > 0, "noise_fir: bad argument");
  RAVE_CHECK_ARG(TS >= 1 && TS <= NF_MAX_TS && NB >= 1 && NB <= NF_MAX_NB && B <= 65535 && C <= 65535,
                 "noise_fir: target_size %d (<= %d) / bands %d (<= %d) outside the kernel's range", TS, NF_MAX_TS, NB,
                 NF_MAX_NB);
  dim3 grid(ceil_div(T, 128), C, B);
  noise_fir_fwd_kernel<<<grid, 128, TS * NB * sizeof(float), (cudaStream_t)stream>>>(h, M, noise, out, C, NB, T, TS);
  RAVE_CHECK_LAUNCH("noise_fir_fwd");
  return 0;
}

extern "C" int rave_noise_fir_bwd(const float *h, const float *M, const float *noise, const float *dout, float *dh,
                                  int B, int C, int NB, int T, int TS, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h && M && noise && dout && dh && B > 0 && C > 0 && T > 0, "noise_fir_bwd: bad argument");
  RAVE_CHECK_ARG(TS >= 1 && TS <= NF_MAX_TS && NB >= 1 && NB <= NF_MAX_NB && B <= 65535 && C <= 65535,
                 "noise_fir_bwd: shape outside the kernel's range");
  dim3 grid(ceil_div(T, 128), C, B);
  noise_fir_bwd_kernel<<<grid, 128, TS * NB * sizeof(float), (cudaStream_t)stream>>>(h, M, noise, dout, dh, C, NB, T, TS);
  RAVE_CHECK_LAUNCH("noise_fir_bwd");
  return 0;
}
