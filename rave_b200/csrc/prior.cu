// The latent prior's own arithmetic (rave/prior/{core,residual_block,model}.py: VariationalPrior.training_step):
//   latent classes : reparametrise -> centre -> PCA -> DiagonalShift -> QuantizedNormal.encode, as class indices
//   embedding      : pre_net (grouped causal conv on the stacked one-hot) as a gather of weight columns, + LeakyReLU
//   gate           : sigmoid(h[:, :C]) * tanh(h[:, C:]) of every ResidualBlock
//   head           : post_net.2 (grouped 1x1) + log-softmax over each group's R logits + cross-entropy against the
//                    class of the next frame; the logits live in shared memory only
// Everything is fp32 CUDA-core arithmetic (these shapes are a few thousand rows) and every sum is added in a fixed order
// (no float atomics): two runs give the same bits.
//
// Streams [B][T][C] are addressed through `cl_bf16`: 1 = the wgmma engine's channel-last layout with bf16 operands,
// 0 = the parity path's [B][C][T] layout in fp32.  Gradients read from a conv's fp32 output (`dg`, `dout`) are fp32
// in both layouts.
#include "common.cuh"

namespace rave {

constexpr int PRIOR_THREADS = 256;
constexpr int PRIOR_MAX_K = 8;        // embedding taps
constexpr int HEAD_P = 16;            // head positions per CTA

__device__ __forceinline__ size_t sidx(bool cl, int b, int t, int c, int T, int C) {
  return cl ? ((size_t)b * T + t) * C + c : ((size_t)b * C + c) * T + t;
}
__device__ __forceinline__ float ldf(const float *p, size_t i) { return p[i]; }
__device__ __forceinline__ float ldf(const __nv_bfloat16 *p, size_t i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void stf(float *p, size_t i, float v) { p[i] = v; }
__device__ __forceinline__ void stf(__nv_bfloat16 *p, size_t i, float v) { p[i] = __float2bfloat16_rn(v); }

// ---------------------------------------------------------------------------------------------------------------------
// classes[b][t'][d] = clamp(floor(R * Phi(y_d(b, t' + D - 1 - d))), 0, R - 1),
//   y_d(b, t) = sum_c pca[d][c] * (eps[b][c][t] * (softplus(scale[b][c][t]) + 1e-4) + mean[b][c][t] - latent_mean[c])
// z = [B][2L][T] (mean | scale), eps [B][L][T].  One thread per output; the per-(b, t, c) sample is recomputed by the D
// threads that read it (L * D multiply-adds per output, a few thousand outputs).
__global__ void __launch_bounds__(PRIOR_THREADS)
prior_latent_classes_kernel(const float *__restrict__ z, const float *__restrict__ eps, const float *__restrict__ lmean,
                            const float *__restrict__ pca, int *__restrict__ cls, int B, int L, int T, int D, int R) {
  const int Tp = T - D + 1;
  const long i = blockIdx.x * (long)PRIOR_THREADS + threadIdx.x;
  if (i >= (long)B * Tp * D) return;
  const int d = (int)(i % D);
  const long n = i / D;
  const int tp = (int)(n % Tp), b = (int)(n / Tp), t = tp + D - 1 - d;
  const float *zm = z + (size_t)b * 2 * L * T + t, *zs = zm + (size_t)L * T, *ep = eps + (size_t)b * L * T + t;
  float acc = 0.f;
  for (int c = 0; c < L; ++c) {
    const float s = centred_sample(zm[(size_t)c * T], zs[(size_t)c * T], ep[(size_t)c * T], lmean[c]);
    acc = fmaf(pca[(size_t)d * L + c], s, acc);
  }
  const float u = 0.5f * (1.f + erff(acc / 1.41421356237309515f));
  int k = (int)floorf(u * (float)R);
  k = k < 0 ? 0 : (k > R - 1 ? R - 1 : k);
  cls[i] = k;
}

// ---------------------------------------------------------------------------------------------------------------------
// pre_net on class indices: group d(o) = o / (Cout / D) reads latent d;
//   x[b][t][o] = LeakyReLU(bias[o] + sum_{k, t + k - (K-1) >= 0} w[o][c_d(b, t + k - (K-1))][k])
// written as the fp32 stream (layout per cl_bf16) and, in bf16 mode, as the channel-last bf16 operand.
__global__ void __launch_bounds__(PRIOR_THREADS)
prior_embed_fwd_kernel(const int *__restrict__ cls, const float *__restrict__ w, const float *__restrict__ bias,
                       float *__restrict__ out, __nv_bfloat16 *__restrict__ op, int B, int Tp, int D, int R, int Cout,
                       int K, int cl, float slope) {
  const long i = blockIdx.x * (long)PRIOR_THREADS + threadIdx.x;
  if (i >= (long)B * Tp * Cout) return;
  const int o = (int)(i % Cout);
  const long n = i / Cout;
  const int t = (int)(n % Tp), b = (int)(n / Tp), d = o / (Cout / D);
  const float *wo = w + (size_t)o * R * K;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) {
    const int s = t + k - (K - 1);
    if (s >= 0) acc += wo[cls[((size_t)b * Tp + s) * D + d] * K + k];
  }
  float v = acc + (bias ? bias[o] : 0.f);
  v = v > 0.f ? v : v * slope;
  out[sidx(cl, b, t, o, Tp, Cout)] = v;
  if (op) op[n * Cout + o] = __float2bfloat16_rn(v);
}

// Its weight gradient, a scatter by class written as a gather: warp = one output channel o, lane = one class r (of a
// 32-class slice, grid.y); every lane walks all B * Tp positions in order and adds dy = dout * LeakyReLU'(x) into the
// taps whose source class is r.  Lane 0 of slice 0 also adds the bias gradient.
template <typename E>
__global__ void __launch_bounds__(PRIOR_THREADS)
prior_embed_wgrad_kernel(const int *__restrict__ cls, const float *__restrict__ dout, const E *__restrict__ x,
                         float *__restrict__ dw, float *__restrict__ dbias, int B, int Tp, int D, int R, int Cout, int K,
                         int cl, float slope) {
  const int o = blockIdx.x * (PRIOR_THREADS / 32) + (threadIdx.x >> 5);
  const int r = blockIdx.y * 32 + (threadIdx.x & 31);
  if (o >= Cout) return;
  const int d = o / (Cout / D);
  float acc[PRIOR_MAX_K];
#pragma unroll
  for (int k = 0; k < PRIOR_MAX_K; ++k) acc[k] = 0.f;
  float accb = 0.f;
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < Tp; ++t) {
      const size_t e = sidx(cl, b, t, o, Tp, Cout);
      const float dy = dout[e] * (ldf(x, e) > 0.f ? 1.f : slope);
      accb += dy;
#pragma unroll
      for (int k = 0; k < PRIOR_MAX_K; ++k) {
        const int s = t + k - (K - 1);
        if (k < K && s >= 0 && cls[((size_t)b * Tp + s) * D + d] == r) acc[k] += dy;
      }
    }
  if (r < R)
#pragma unroll
    for (int k = 0; k < PRIOR_MAX_K; ++k)
      if (k < K) dw[((size_t)o * R + r) * K + k] = acc[k];
  if (dbias && r == 0) dbias[o] = accb;
}

// ---------------------------------------------------------------------------------------------------------------------
// gated unit of ResidualBlock: g = sigmoid(h[:, c]) * tanh(h[:, C + c]), h [B][T][2C] / g [B][T][C] (layout per cl)
template <typename E>
__global__ void __launch_bounds__(PRIOR_THREADS)
gate_fwd_kernel(const E *__restrict__ h, E *__restrict__ g, int B, int C, int T, int cl) {
  const long i = blockIdx.x * (long)PRIOR_THREADS + threadIdx.x;
  if (i >= (long)B * T * C) return;
  int b, t, c;
  if (cl) { c = (int)(i % C); const long n = i / C; t = (int)(n % T); b = (int)(n / T); }
  else { t = (int)(i % T); const long n = i / T; c = (int)(n % C); b = (int)(n / C); }
  const float a = ldf(h, sidx(cl, b, t, c, T, 2 * C)), v = ldf(h, sidx(cl, b, t, C + c, T, 2 * C));
  stf(g, sidx(cl, b, t, c, T, C), (1.f / (1.f + expf(-a))) * tanhf(v));
}

// dh[:, c] = dg * tanh(h_b) * s (1 - s),  dh[:, C + c] = dg * s * (1 - tanh(h_b)^2),  s = sigmoid(h_a)
template <typename E>
__global__ void __launch_bounds__(PRIOR_THREADS)
gate_bwd_kernel(const float *__restrict__ dg, const E *__restrict__ h, E *__restrict__ dh, int B, int C, int T, int cl) {
  const long i = blockIdx.x * (long)PRIOR_THREADS + threadIdx.x;
  if (i >= (long)B * T * C) return;
  int b, t, c;
  if (cl) { c = (int)(i % C); const long n = i / C; t = (int)(n % T); b = (int)(n / T); }
  else { t = (int)(i % T); const long n = i / T; c = (int)(n % C); b = (int)(n / C); }
  const size_t ea = sidx(cl, b, t, c, T, 2 * C), eb = sidx(cl, b, t, C + c, T, 2 * C);
  const float s = 1.f / (1.f + expf(-ldf(h, ea))), th = tanhf(ldf(h, eb)), gv = dg[sidx(cl, b, t, c, T, C)];
  stf(dh, ea, gv * th * s * (1.f - s));
  stf(dh, eb, gv * s * (1.f - th * th));
}

// ---------------------------------------------------------------------------------------------------------------------
// Head.  CTA (chunk, d) owns HEAD_P consecutive positions n = b * Tp + t of group d.  The input is x = LeakyReLU(p)
// of post_net.0's output p [B][Tp][Cin] (group d: channels d * Cg .. + Cg, Cg = Cin / D); the logits
//   l[n][r] = sum_j w[d R + r][j] x[n][d Cg + j] + bias[d R + r]
// stay in shared memory.  A position has a target (the class of the next frame, cls[b][t + 1][d]) when t < Tp - 1.
// Shared memory: w [R][Cg], bias [R], xs [P][Cg], lg [P][R], lse [P].
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename E>
__device__ void head_logits(const E *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                            float *sw, float *sb, float *xs, float *lg, float *lse, int n0, int d, int B, int Tp, int R,
                            int Cin, int Cg, int cl, float slope) {
  const int tid = threadIdx.x, N = B * Tp;
  for (int e = tid; e < R * Cg; e += PRIOR_THREADS) sw[e] = w[(size_t)d * R * Cg + e];
  for (int e = tid; e < R; e += PRIOR_THREADS) sb[e] = bias ? bias[d * R + e] : 0.f;
  for (int e = tid; e < HEAD_P * Cg; e += PRIOR_THREADS) {
    const int p = e / Cg, j = e % Cg, n = n0 + p;
    float v = 0.f;
    if (n < N) {
      v = ldf(x, sidx(cl, n / Tp, n % Tp, d * Cg + j, Tp, Cin));
      v = v > 0.f ? v : v * slope;
    }
    xs[e] = v;
  }
  __syncthreads();
  for (int e = tid; e < HEAD_P * R; e += PRIOR_THREADS) {
    const int p = e / R, r = e % R;
    const float *wr = sw + r * Cg, *xp = xs + p * Cg;
    float acc = 0.f;
    for (int j = 0; j < Cg; ++j) acc = fmaf(wr[j], xp[j], acc);
    lg[e] = acc + sb[r];
  }
  __syncthreads();
  // log-sum-exp per position: warp w takes positions w, w + 8
  const int warp = tid >> 5, lane = tid & 31;
  for (int p = warp; p < HEAD_P; p += PRIOR_THREADS / 32) {
    float m = -INFINITY;
    for (int r = lane; r < R; r += 32) m = fmaxf(m, lg[p * R + r]);
    m = warp_max(m);
    float s = 0.f;
    for (int r = lane; r < R; r += 32) s += expf(lg[p * R + r] - m);
    s = warp_sum(s);
    if (lane == 0) lse[p] = m + logf(s);
  }
  __syncthreads();
}

__host__ __device__ inline size_t head_smem_floats(int R, int Cg) {
  return (size_t)R * Cg + R + (size_t)HEAD_P * Cg + (size_t)HEAD_P * R + HEAD_P;
}

// part[chunk * D + d] = sum over the CTA's positions with a target of (lse - l[target]), in position order
template <typename E>
__global__ void __launch_bounds__(PRIOR_THREADS)
head_ce_fwd_kernel(const E *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                   const int *__restrict__ cls, float *__restrict__ part, int B, int Tp, int D, int R, int Cin, int cl,
                   float slope) {
  extern __shared__ float smem[];
  const int Cg = Cin / D, d = blockIdx.y, n0 = blockIdx.x * HEAD_P;
  float *sw = smem, *sb = sw + R * Cg, *xs = sb + R, *lg = xs + HEAD_P * Cg, *lse = lg + HEAD_P * R;
  head_logits(x, w, bias, sw, sb, xs, lg, lse, n0, d, B, Tp, R, Cin, Cg, cl, slope);
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int p = 0; p < HEAD_P; ++p) {
      const int n = n0 + p, t = n % Tp;
      if (n < B * Tp && t < Tp - 1) s += lse[p] - lg[p * R + cls[((size_t)n + 1) * D + d]];
    }
    part[(size_t)blockIdx.x * D + d] = s;
  }
}

// dl = g * inv_count * (softmax(l) - onehot(target)) (0 without a target);  dx = (W_d^T dl) * LeakyReLU'(p);
// part[chunk][d][r][0..Cg) = sum_p dl[p][r] x[p][j], part[chunk][d][r][Cg] = sum_p dl[p][r]
template <typename E>
__global__ void __launch_bounds__(PRIOR_THREADS)
head_ce_bwd_kernel(const E *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                   const int *__restrict__ cls, const float *__restrict__ gloss, E *__restrict__ dx,
                   float *__restrict__ part, int B, int Tp, int D, int R, int Cin, int cl, float slope, float inv_count) {
  extern __shared__ float smem[];
  const int Cg = Cin / D, d = blockIdx.y, n0 = blockIdx.x * HEAD_P, N = B * Tp, tid = threadIdx.x;
  float *sw = smem, *sb = sw + R * Cg, *xs = sb + R, *lg = xs + HEAD_P * Cg, *lse = lg + HEAD_P * R;
  head_logits(x, w, bias, sw, sb, xs, lg, lse, n0, d, B, Tp, R, Cin, Cg, cl, slope);
  const float gs = gloss[0] * inv_count;
  for (int e = tid; e < HEAD_P * R; e += PRIOR_THREADS) {
    const int p = e / R, r = e % R, n = n0 + p;
    float v = 0.f;
    if (n < N && n % Tp < Tp - 1) {
      const int tgt = cls[((size_t)n + 1) * D + d];
      v = gs * (expf(lg[e] - lse[p]) - (r == tgt ? 1.f : 0.f));
    }
    lg[e] = v;
  }
  __syncthreads();
  for (int e = tid; e < HEAD_P * Cg; e += PRIOR_THREADS) {
    const int p = e / Cg, j = e % Cg, n = n0 + p;
    if (n >= N) continue;
    float s = 0.f;
    for (int r = 0; r < R; ++r) s = fmaf(lg[p * R + r], sw[r * Cg + j], s);
    const size_t ei = sidx(cl, n / Tp, n % Tp, d * Cg + j, Tp, Cin);
    stf(dx, ei, ldf(x, ei) > 0.f ? s : s * slope);
  }
  float *pd = part + ((size_t)blockIdx.x * D + d) * R * (Cg + 1);
  for (int e = tid; e < R * (Cg + 1); e += PRIOR_THREADS) {
    const int r = e / (Cg + 1), j = e % (Cg + 1);
    float s = 0.f;
    for (int p = 0; p < HEAD_P; ++p) s = fmaf(lg[p * R + r], j < Cg ? xs[p * Cg + j] : 1.f, s);
    pd[e] = s;
  }
}

// dw[(d R + r) Cg + j] / dbias[d R + r] = the chunks' partials added in chunk order
__global__ void __launch_bounds__(PRIOR_THREADS)
head_ce_wreduce_kernel(const float *__restrict__ part, float *__restrict__ dw, float *__restrict__ dbias, int chunks,
                       int D, int R, int Cg) {
  const long per = (long)D * R * (Cg + 1);
  const long e = blockIdx.x * (long)PRIOR_THREADS + threadIdx.x;
  if (e >= per) return;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += part[(size_t)c * per + e];
  const long dr = e / (Cg + 1);
  const int j = (int)(e % (Cg + 1));
  if (j < Cg) dw[dr * Cg + j] = s;
  else if (dbias) dbias[dr] = s;
}

// loss[0] = inv_count * sum of the n partials: fixed per-thread strides, then a fixed-order tree
__global__ void __launch_bounds__(PRIOR_THREADS)
sum_scale_kernel(const float *__restrict__ part, float *__restrict__ out, long n, float scale) {
  __shared__ float red[PRIOR_THREADS];
  float s = 0.f;
  for (long i = threadIdx.x; i < n; i += PRIOR_THREADS) s += part[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = PRIOR_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = red[0] * scale;
}

inline int blocks_for(long n) { return (int)((n + PRIOR_THREADS - 1) / PRIOR_THREADS); }

template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024 &&
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) {
    set_error("prior head: %zu bytes of shared memory refused", bytes);
    return 2;
  }
  return 0;
}

}  // namespace rave

using rave::PRIOR_THREADS;

extern "C" int rave_prior_latent_classes(const float *z, const float *eps, const float *latent_mean,
                                         const float *latent_pca, int *classes, int B, int L, int T, int D, int R,
                                         void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && eps && latent_mean && latent_pca && classes, "prior_latent_classes: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && D > 0 && D <= L && T >= D && R > 0,
                 "prior_latent_classes: bad shape (B %d, L %d, T %d, D %d, R %d)", B, L, T, D, R);
  const long n = (long)B * (T - D + 1) * D;
  prior_latent_classes_kernel<<<blocks_for(n), PRIOR_THREADS, 0, (cudaStream_t)stream>>>(z, eps, latent_mean,
                                                                                          latent_pca, classes, B, L, T,
                                                                                          D, R);
  RAVE_CHECK_LAUNCH("prior_latent_classes");
  return 0;
}

extern "C" int rave_prior_embed_fwd(const int *classes, const float *w, const float *bias, float *out_f32,
                                    void *out_op_bf16, int B, int Tp, int D, int R, int Cout, int K, int cl_bf16,
                                    float slope, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(classes && w && out_f32 && (cl_bf16 || !out_op_bf16), "prior_embed_fwd: bad pointer");
  RAVE_CHECK_ARG(B > 0 && Tp > 0 && D > 0 && R > 0 && K > 0 && Cout > 0 && Cout % D == 0,
                 "prior_embed_fwd: bad shape (Cout %d, D %d)", Cout, D);
  const long n = (long)B * Tp * Cout;
  prior_embed_fwd_kernel<<<blocks_for(n), PRIOR_THREADS, 0, (cudaStream_t)stream>>>(
      classes, w, bias, out_f32, (__nv_bfloat16 *)out_op_bf16, B, Tp, D, R, Cout, K, cl_bf16 != 0, slope);
  RAVE_CHECK_LAUNCH("prior_embed_fwd");
  return 0;
}

extern "C" int rave_prior_embed_wgrad(const int *classes, const float *dout, const void *x, float *dw, float *dbias,
                                      int B, int Tp, int D, int R, int Cout, int K, int cl_bf16, float slope,
                                      void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(classes && dout && x && dw, "prior_embed_wgrad: null pointer");
  RAVE_CHECK_ARG(B > 0 && Tp > 0 && D > 0 && R > 0 && K > 0 && K <= PRIOR_MAX_K && Cout > 0 && Cout % D == 0,
                 "prior_embed_wgrad: bad shape (Cout %d, D %d, K %d <= %d)", Cout, D, K, PRIOR_MAX_K);
  const dim3 grid(ceil_div(Cout, PRIOR_THREADS / 32), ceil_div(R, 32));
  const cudaStream_t s = (cudaStream_t)stream;
  if (cl_bf16)
    prior_embed_wgrad_kernel<<<grid, PRIOR_THREADS, 0, s>>>(classes, dout, (const __nv_bfloat16 *)x, dw, dbias, B, Tp,
                                                             D, R, Cout, K, 1, slope);
  else
    prior_embed_wgrad_kernel<<<grid, PRIOR_THREADS, 0, s>>>(classes, dout, (const float *)x, dw, dbias, B, Tp, D, R,
                                                             Cout, K, 0, slope);
  RAVE_CHECK_LAUNCH("prior_embed_wgrad");
  return 0;
}

extern "C" int rave_gate_fwd(const void *h, void *g, int B, int C, int T, int cl_bf16, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h && g && B > 0 && C > 0 && T > 0, "gate_fwd: bad argument");
  const long n = (long)B * T * C;
  const cudaStream_t s = (cudaStream_t)stream;
  if (cl_bf16)
    gate_fwd_kernel<<<blocks_for(n), PRIOR_THREADS, 0, s>>>((const __nv_bfloat16 *)h, (__nv_bfloat16 *)g, B, C, T, 1);
  else
    gate_fwd_kernel<<<blocks_for(n), PRIOR_THREADS, 0, s>>>((const float *)h, (float *)g, B, C, T, 0);
  RAVE_CHECK_LAUNCH("gate_fwd");
  return 0;
}

extern "C" int rave_gate_bwd(const float *dg, const void *h, void *dh, int B, int C, int T, int cl_bf16,
                             void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dg && h && dh && B > 0 && C > 0 && T > 0, "gate_bwd: bad argument");
  const long n = (long)B * T * C;
  const cudaStream_t s = (cudaStream_t)stream;
  if (cl_bf16)
    gate_bwd_kernel<<<blocks_for(n), PRIOR_THREADS, 0, s>>>(dg, (const __nv_bfloat16 *)h, (__nv_bfloat16 *)dh, B, C, T,
                                                             1);
  else
    gate_bwd_kernel<<<blocks_for(n), PRIOR_THREADS, 0, s>>>(dg, (const float *)h, (float *)dh, B, C, T, 0);
  RAVE_CHECK_LAUNCH("gate_bwd");
  return 0;
}

static int head_check(const void *x, const float *w, const int *cls, int B, int Tp, int D, int R, int Cin) {
  RAVE_CHECK_ARG(x && w && cls, "prior_head_ce: null pointer");
  RAVE_CHECK_ARG(B > 0 && Tp > 1 && D > 0 && R > 0 && Cin > 0 && Cin % D == 0,
                 "prior_head_ce: bad shape (B %d, Tp %d, D %d, R %d, Cin %d)", B, Tp, D, R, Cin);
  RAVE_CHECK_ARG(rave::head_smem_floats(R, Cin / D) * 4 <= 200 * 1024, "prior_head_ce: R * Cin / D too large");
  return 0;
}

extern "C" int rave_prior_head_ce_fwd(const void *x, const float *w, const float *bias, const int *classes, float *loss,
                                      int B, int Tp, int D, int R, int Cin, int cl_bf16, float slope, void *stream) {
  using namespace rave;
  if (int rc = head_check(x, w, classes, B, Tp, D, R, Cin)) return rc;
  RAVE_CHECK_ARG(loss, "prior_head_ce_fwd: null loss");
  const cudaStream_t s = (cudaStream_t)stream;
  const int chunks = ceil_div(B * Tp, HEAD_P);
  const size_t smem = head_smem_floats(R, Cin / D) * sizeof(float);
  float *part = nullptr;
  if (cudaMallocAsync((void **)&part, (size_t)chunks * D * sizeof(float), s) != cudaSuccess) {
    set_error("prior_head_ce_fwd: cudaMallocAsync failed");
    return 2;
  }
  const dim3 grid(chunks, D);
  int rc = 0;
  if (cl_bf16) {
    if (!(rc = set_smem(head_ce_fwd_kernel<__nv_bfloat16>, smem)))
      head_ce_fwd_kernel<<<grid, PRIOR_THREADS, smem, s>>>((const __nv_bfloat16 *)x, w, bias, classes, part, B, Tp, D, R,
                                                           Cin, 1, slope);
  } else {
    if (!(rc = set_smem(head_ce_fwd_kernel<float>, smem)))
      head_ce_fwd_kernel<<<grid, PRIOR_THREADS, smem, s>>>((const float *)x, w, bias, classes, part, B, Tp, D, R, Cin,
                                                           0, slope);
  }
  if (!rc) {
    const double count = (double)B * D * (Tp - 1);
    sum_scale_kernel<<<1, PRIOR_THREADS, 0, s>>>(part, loss, (long)chunks * D, (float)(1.0 / count));
  }
  cudaFreeAsync(part, s);
  if (rc) return rc;
  RAVE_CHECK_LAUNCH("prior_head_ce_fwd");
  return 0;
}

extern "C" int rave_prior_head_ce_bwd(const void *x, const float *w, const float *bias, const int *classes,
                                      const float *gloss, void *dx, float *dw, float *dbias, int B, int Tp, int D, int R,
                                      int Cin, int cl_bf16, float slope, void *stream) {
  using namespace rave;
  if (int rc = head_check(x, w, classes, B, Tp, D, R, Cin)) return rc;
  RAVE_CHECK_ARG(gloss && dx && dw, "prior_head_ce_bwd: null pointer");
  const cudaStream_t s = (cudaStream_t)stream;
  const int chunks = ceil_div(B * Tp, HEAD_P), Cg = Cin / D;
  const size_t smem = head_smem_floats(R, Cg) * sizeof(float);
  const long per = (long)D * R * (Cg + 1);
  float *part = nullptr;
  if (cudaMallocAsync((void **)&part, (size_t)chunks * per * sizeof(float), s) != cudaSuccess) {
    set_error("prior_head_ce_bwd: cudaMallocAsync failed");
    return 2;
  }
  const dim3 grid(chunks, D);
  const float inv_count = (float)(1.0 / ((double)B * D * (Tp - 1)));
  int rc = 0;
  if (cl_bf16) {
    if (!(rc = set_smem(head_ce_bwd_kernel<__nv_bfloat16>, smem)))
      head_ce_bwd_kernel<<<grid, PRIOR_THREADS, smem, s>>>((const __nv_bfloat16 *)x, w, bias, classes, gloss,
                                                           (__nv_bfloat16 *)dx, part, B, Tp, D, R, Cin, 1, slope,
                                                           inv_count);
  } else {
    if (!(rc = set_smem(head_ce_bwd_kernel<float>, smem)))
      head_ce_bwd_kernel<<<grid, PRIOR_THREADS, smem, s>>>((const float *)x, w, bias, classes, gloss, (float *)dx, part,
                                                           B, Tp, D, R, Cin, 0, slope, inv_count);
  }
  if (!rc) head_ce_wreduce_kernel<<<blocks_for(per), PRIOR_THREADS, 0, s>>>(part, dw, dbias, chunks, D, R, Cg);
  cudaFreeAsync(part, s);
  if (rc) return rc;
  RAVE_CHECK_LAUNCH("prior_head_ce_bwd");
  return 0;
}
