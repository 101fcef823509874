// Weight norm, stand-alone activations and the generator tail.
//
// Reference: torch.nn.utils.weight_norm via blocks.normalization (rave/blocks.py:15-22);
// Snake (blocks.py:852-860); LeakyReLU(.2) (blocks.py:56,90,528,614); GeneratorV2 tail
// x * sigmoid(a) -> tanh (blocks.py:704-711).
#include "common.cuh"

namespace rave {

__device__ __forceinline__ float block_reduce_sum(float v, float *red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (wid == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if (lane == 0) red[0] = r;
  }
  __syncthreads();
  return red[0];
}

// one CTA per leading index c0
__global__ void __launch_bounds__(256)
weight_norm_fwd_kernel(const float *__restrict__ v, const float *__restrict__ g, float *__restrict__ w,
                       float *__restrict__ norm_out, int R) {
  __shared__ float red[32];
  const int c = blockIdx.x;
  const float *vr = v + (size_t)c * R;
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    float x = vr[i];
    s = fmaf(x, x, s);
  }
  const float n = sqrtf(block_reduce_sum(s, red));
  const float scale = g[c] / n;
  for (int i = threadIdx.x; i < R; i += blockDim.x) w[(size_t)c * R + i] = vr[i] * scale;
  if (threadIdx.x == 0 && norm_out) norm_out[c] = n;
}

__global__ void __launch_bounds__(256)
weight_norm_bwd_kernel(const float *__restrict__ dw, const float *__restrict__ v,
                       const float *__restrict__ g, const float *__restrict__ norm,
                       float *__restrict__ dv, float *__restrict__ dg, int R) {
  __shared__ float red[32];
  const int c = blockIdx.x;
  const float *vr = v + (size_t)c * R;
  const float *dr = dw + (size_t)c * R;
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += blockDim.x) s = fmaf(dr[i], vr[i], s);
  const float dot = block_reduce_sum(s, red);
  const float n = norm[c];
  const float gn = g[c] / n;
  const float coef = dot / (n * n);
  for (int i = threadIdx.x; i < R; i += blockDim.x) dv[(size_t)c * R + i] = gn * (dr[i] - vr[i] * coef);
  if (threadIdx.x == 0) dg[c] = dot / n;
}

// grid: (ceil(L/1024), C, B)
__global__ void __launch_bounds__(256)
act_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int C, int L, int act, float slope,
               const float *__restrict__ alpha) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float al = (act == RAVE_ACT_SNAKE) ? alpha[c] : 0.f;
  const size_t base = ((size_t)b * C + c) * L;
  for (int t = blockIdx.x * 1024 + threadIdx.x; t < min(L, (int)(blockIdx.x + 1) * 1024); t += 256)
    y[base + t] = act_apply(x[base + t], act, slope, al);
}

// dx = dy * act'(x); Snake: dalpha[c] += sum dy * d/dalpha  (block-order sum over CTAs; dalpha pre-zeroed)
__global__ void __launch_bounds__(256)
act_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ x, float *__restrict__ dx,
               float *__restrict__ dalpha, int C, int L, int act, float slope,
               const float *__restrict__ alpha, const BlockSum bs) {
  __shared__ float red[32];
  const int c = blockIdx.y, b = blockIdx.z;
  const float al = (act == RAVE_ACT_SNAKE) ? alpha[c] : 0.f;
  const size_t base = ((size_t)b * C + c) * L;
  float s = 0.f;
  for (int t = blockIdx.x * 1024 + threadIdx.x; t < min(L, (int)(blockIdx.x + 1) * 1024); t += 256) {
    const float xv = x[base + t], g = dy[base + t];
    dx[base + t] = g * act_grad(xv, act, slope, al);
    if (act == RAVE_ACT_SNAKE) {
      // d/dalpha [ sin^2(a x) / (a + eps) ] = x sin(2 a x)/(a+eps) - sin^2(a x)/(a+eps)^2
      const float ae = al + 1e-9f;
      const float sn = sinf(al * xv);
      s += g * (xv * sinf(2.f * al * xv) / ae - sn * sn / (ae * ae));
    }
  }
  if (act == RAVE_ACT_SNAKE && dalpha) {      // uniform over the grid
    const float tot = block_reduce_sum(s, red);
    if (threadIdx.x == 0) block_sum_put(bs, 0, tot);
    block_sum_finish(bs, dalpha);             // one group per channel (grid y)
  }
}

// Activations without a per-channel parameter (LeakyReLU) do not care about the [B][C][L] shape: flat 16-byte passes
// (the Descript discriminator's channel-last features have L = 32: one (b, c) row per CTA used 32 of 256 threads).
__global__ void __launch_bounds__(256)
act_flat_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, long n, int act, float slope, int vec) {
  const long n4 = vec ? (n >> 2) : 0;
  const float4 *x4 = reinterpret_cast<const float4 *>(x);
  float4 *y4 = reinterpret_cast<float4 *>(y);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n4; i += (long)gridDim.x * 256) {
    float4 a = __ldg(x4 + i);
    a.x = act_apply(a.x, act, slope, 0.f); a.y = act_apply(a.y, act, slope, 0.f);
    a.z = act_apply(a.z, act, slope, 0.f); a.w = act_apply(a.w, act, slope, 0.f);
    y4[i] = a;
  }
  for (long i = (n4 << 2) + blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256)
    y[i] = act_apply(x[i], act, slope, 0.f);
}

__global__ void __launch_bounds__(256)
act_flat_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ x, float *__restrict__ dx, long n, int act,
                    float slope, int vec) {
  const long n4 = vec ? (n >> 2) : 0;
  const float4 *x4 = reinterpret_cast<const float4 *>(x), *g4 = reinterpret_cast<const float4 *>(dy);
  float4 *d4 = reinterpret_cast<float4 *>(dx);
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n4; i += (long)gridDim.x * 256) {
    const float4 a = __ldg(x4 + i), g = __ldg(g4 + i);
    d4[i] = make_float4(g.x * act_grad(a.x, act, slope, 0.f), g.y * act_grad(a.y, act, slope, 0.f),
                        g.z * act_grad(a.z, act, slope, 0.f), g.w * act_grad(a.w, act, slope, 0.f));
  }
  for (long i = (n4 << 2) + blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256)
    dx[i] = dy[i] * act_grad(x[i], act, slope, 0.f);
}

// y[b][c][t] = tanh(x[b][c][t] * sigmoid(x[b][C+c][t]))
__global__ void __launch_bounds__(256)
am_tanh_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int C, int L, long total) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const long bc = i / L;
    const int t = (int)(i - bc * L);
    const int b = (int)(bc / C), c = (int)(bc - (long)b * C);
    const size_t xo = ((size_t)b * 2 * C + c) * L + t;
    const float w = x[xo], a = x[xo + (size_t)C * L];
    const float sg = 1.f / (1.f + expf(-a));
    y[i] = tanhf(w * sg);
  }
}

__global__ void __launch_bounds__(256)
am_tanh_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ x, float *__restrict__ dx,
                   int C, int L, long total) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const long bc = i / L;
    const int t = (int)(i - bc * L);
    const int b = (int)(bc / C), c = (int)(bc - (long)b * C);
    const size_t xo = ((size_t)b * 2 * C + c) * L + t;
    const float w = x[xo], a = x[xo + (size_t)C * L];
    const float sg = 1.f / (1.f + expf(-a));
    const float th = tanhf(w * sg);
    const float g = dy[i] * (1.f - th * th);
    dx[xo] = g * sg;
    dx[xo + (size_t)C * L] = g * w * sg * (1.f - sg);
  }
}

// VariationalEncoder.reparametrize (rave/blocks.py:725-737), one pass: z [B][2C][L] = (mean | scale),
//   std = softplus(scale) + 1e-4, zs = eps * std + mean, kl_sum += sum (mean^2 + std^2 - log(std^2) - 1)
// (the reference's ~14 elementwise / reduction launches on a 0.26 M element tensor).  kl_sum must be zeroed by the caller.
__global__ void __launch_bounds__(256)
reparam_fwd_kernel(const float *__restrict__ z, const float *__restrict__ eps, float *__restrict__ zs,
                   float *__restrict__ kl_sum, long CL, long total, const BlockSum bs) {
  __shared__ float red[32];
  float acc = 0.f;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const long b = i / CL;
    const long zo = i + b * CL;                       // b * 2CL + (i - b * CL)
    const float mean = z[zo], scale = z[zo + CL];
    const float sp = scale > 20.f ? scale : log1pf(expf(scale));      // F.softplus (beta 1, threshold 20)
    const float sd = sp + 1e-4f;
    const float var = sd * sd;
    zs[i] = eps[i] * sd + mean;
    acc += mean * mean + var - logf(var) - 1.f;
  }
  const float tot = block_reduce_sum(acc, red);
  if (threadIdx.x == 0) block_sum_put(bs, 0, tot);
  block_sum_finish(bs, kl_sum);
}

// y = bf16(act(x)); grid (ceil(L/2048), C, B), 2 elements per thread-iteration
__global__ void __launch_bounds__(256)
act_to_bf16_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ y, int C, int L, int act,
                   float slope, const float *__restrict__ alpha) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float al = (act == RAVE_ACT_SNAKE) ? alpha[c] : 0.f;
  const size_t base = ((size_t)b * C + c) * L;
  const int t_end = min(L, (int)(blockIdx.x + 1) * 2048);
  for (int t = blockIdx.x * 2048 + threadIdx.x; t < t_end; t += 256)
    y[base + t] = __float2bfloat16_rn(act_apply(x[base + t], act, slope, al));
}

// w[Cout][Cin][K] (transpose=0) or w[Cin][Cout][K] (transpose=1) -> wt[K][Cout][Cin] bf16;
// flip=1 reverses the tap order (dgrad of a stride-1 conv is a conv with flipped taps).
__global__ void __launch_bounds__(256)
weight_tapmajor_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wt, int Cout, int Cin,
                       int K, int transpose, int flip) {
  const long total = (long)K * Cout * Cin;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int ci = (int)(i % Cin);
    const long r = i / Cin;
    const int co = (int)(r % Cout);
    const int k = (int)(r / Cout);
    const int ks = flip ? (K - 1 - k) : k;
    const size_t src = transpose ? ((size_t)ci * Cout + co) * K + ks : ((size_t)co * Cin + ci) * K + ks;
    wt[i] = __float2bfloat16_rn(w[src]);
  }
}

}  // namespace rave

extern "C" int rave_weight_norm_fwd(const float *v, const float *g, float *w, float *norm_out, int C0,
                                    int R, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(v && g && w, "weight_norm_fwd: null pointer");
  RAVE_CHECK_ARG(C0 > 0 && R > 0, "weight_norm_fwd: bad shape");
  weight_norm_fwd_kernel<<<C0, 256, 0, (cudaStream_t)stream>>>(v, g, w, norm_out, R);
  RAVE_CHECK_LAUNCH("weight_norm_fwd");
  return 0;
}

extern "C" int rave_weight_norm_bwd(const float *dw, const float *v, const float *g, const float *norm,
                                    float *dv, float *dg, int C0, int R, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dw && v && g && norm && dv && dg, "weight_norm_bwd: null pointer");
  RAVE_CHECK_ARG(C0 > 0 && R > 0, "weight_norm_bwd: bad shape");
  weight_norm_bwd_kernel<<<C0, 256, 0, (cudaStream_t)stream>>>(dw, v, g, norm, dv, dg, R);
  RAVE_CHECK_LAUNCH("weight_norm_bwd");
  return 0;
}

extern "C" int rave_act_fwd(const float *x, float *y, int B, int C, int L, int act, float slope,
                            const float *alpha, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && y, "act_fwd: null pointer");
  RAVE_CHECK_ARG(B > 0 && C > 0 && L > 0 && B <= 65535 && C <= 65535, "act_fwd: bad shape");
  RAVE_CHECK_ARG(act != RAVE_ACT_SNAKE || alpha, "act_fwd: snake needs alpha");
  if (act != RAVE_ACT_SNAKE) {
    const long n = (long)B * C * L;
    const int vec = (((uintptr_t)x | (uintptr_t)y) & 15) == 0;
    long blocks = ((vec ? n / 4 : n) + 255) / 256;
    blocks = blocks < 1 ? 1 : (blocks > 132 * 16 ? 132 * 16 : blocks);
    act_flat_fwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, n, act, slope, vec);
    RAVE_CHECK_LAUNCH("act_fwd");
    return 0;
  }
  dim3 grid(ceil_div(L, 1024), C, B);
  act_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, C, L, act, slope, alpha);
  RAVE_CHECK_LAUNCH("act_fwd");
  return 0;
}

extern "C" int rave_act_bwd(const float *dy, const float *x, float *dx, float *dalpha, int B, int C,
                            int L, int act, float slope, const float *alpha, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dy && x && dx, "act_bwd: null pointer");
  RAVE_CHECK_ARG(B > 0 && C > 0 && L > 0 && B <= 65535 && C <= 65535, "act_bwd: bad shape");
  RAVE_CHECK_ARG(act != RAVE_ACT_SNAKE || alpha, "act_bwd: snake needs alpha");
  if (act != RAVE_ACT_SNAKE) {
    const long n = (long)B * C * L;
    const int vec = (((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dx) & 15) == 0;
    long blocks = ((vec ? n / 4 : n) + 255) / 256;
    blocks = blocks < 1 ? 1 : (blocks > 132 * 16 ? 132 * 16 : blocks);
    act_flat_bwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(dy, x, dx, n, act, slope, vec);
    RAVE_CHECK_LAUNCH("act_bwd");
    return 0;
  }
  if (act == RAVE_ACT_SNAKE && dalpha) cudaMemsetAsync(dalpha, 0, sizeof(float) * C, (cudaStream_t)stream);
  dim3 grid(ceil_div(L, 1024), C, B);
  BlockSum bs;
  memset(&bs, 0, sizeof(bs));
  if (dalpha)
    if (int rc = block_sum_begin(&bs, (long)grid.x * grid.y * grid.z, 1, (cudaStream_t)stream, 1)) return rc;
  act_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dy, x, dx, dalpha, C, L, act, slope, alpha, bs);
  if (dalpha) block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("act_bwd");
  return 0;
}

extern "C" int rave_am_tanh_fwd(const float *x, float *y, int B, int C, int L, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && y && B > 0 && C > 0 && L > 0, "am_tanh_fwd: bad argument");
  const long total = (long)B * C * L;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  am_tanh_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, y, C, L, total);
  RAVE_CHECK_LAUNCH("am_tanh_fwd");
  return 0;
}

extern "C" int rave_am_tanh_bwd(const float *dy, const float *x, float *dx, int B, int C, int L,
                                void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dy && x && dx && B > 0 && C > 0 && L > 0, "am_tanh_bwd: bad argument");
  const long total = (long)B * C * L;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  am_tanh_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dy, x, dx, C, L, total);
  RAVE_CHECK_LAUNCH("am_tanh_bwd");
  return 0;
}

extern "C" int rave_reparam_fwd(const float *z, const float *eps, float *zs, float *kl_sum, int B, int C, int L,
                                void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && eps && zs && kl_sum && B > 0 && C > 0 && L > 0, "reparam_fwd: bad argument");
  const long total = (long)B * C * L;
  int blocks = (int)((total + 1023) / 1024);            // ~4 elements per thread: few partials, still every SM busy
  if (blocks > 132 * 4) blocks = 132 * 4;
  if (blocks < 1) blocks = 1;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, blocks, 1, (cudaStream_t)stream)) return rc;
  reparam_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(z, eps, zs, kl_sum, (long)C * L, total, bs);
  block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("reparam_fwd");
  return 0;
}

extern "C" int rave_act_to_bf16(const float *x, void *y_bf16, int B, int C, int L, int act, float slope,
                                const float *alpha, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && y_bf16, "act_to_bf16: null pointer");
  RAVE_CHECK_ARG(B > 0 && C > 0 && L > 0 && B <= 65535 && C <= 65535, "act_to_bf16: bad shape");
  RAVE_CHECK_ARG(act != RAVE_ACT_SNAKE || alpha, "act_to_bf16: snake needs alpha");
  dim3 grid(ceil_div(L, 2048), C, B);
  act_to_bf16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16 *)y_bf16, C, L, act, slope,
                                                            alpha);
  RAVE_CHECK_LAUNCH("act_to_bf16");
  return 0;
}

extern "C" int rave_weight_to_tapmajor_bf16(const float *w, void *wt_bf16, int Cout, int Cin, int K,
                                            int transpose, int flip, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(w && wt_bf16 && Cout > 0 && Cin > 0 && K > 0, "weight_to_tapmajor: bad argument");
  const long total = (long)K * Cout * Cin;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  weight_tapmajor_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__nv_bfloat16 *)wt_bf16, Cout, Cin,
                                                                  K, transpose, flip);
  RAVE_CHECK_LAUNCH("weight_to_tapmajor");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// layout converters: module-boundary [B][C][L] fp32  <->  engine channel-last [B][L][C]
// 32x32 tiles through shared memory so both sides are coalesced.
// ---------------------------------------------------------------------------------------------
namespace rave {

// grid: (ceil(L/32), ceil(C/32), B), block (32, 8)
__global__ void __launch_bounds__(256)
ncl_to_cl_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ yb, float *__restrict__ yf, int C,
                 int L, int act, float slope, const float *__restrict__ alpha) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, l = l0 + tx;
    tile[ty + 8 * i][tx] = (c < C && l < L) ? x[((size_t)b * C + c) * L + l] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + 8 * i, c = c0 + tx;
    if (l < L && c < C) {
      const float v = tile[tx][ty + 8 * i];
      const size_t o = ((size_t)b * L + l) * C + c;
      if (yf) yf[o] = v;
      if (yb) yb[o] = __float2bfloat16_rn(act_apply(v, act, slope, act == RAVE_ACT_SNAKE ? alpha[c] : 0.f));
    }
  }
}

// x3 operand entry: y[b][l][0..C) = bf16(x), y[b][l][C..2C) = bf16(x - hi)
__global__ void __launch_bounds__(256)
ncl_to_cl_x3_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ y, int C, int L) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, l = l0 + tx;
    tile[ty + 8 * i][tx] = (c < C && l < L) ? x[((size_t)b * C + c) * L + l] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + 8 * i, c = c0 + tx;
    if (l < L && c < C) {
      const float v = tile[tx][ty + 8 * i];
      const size_t o = ((size_t)b * L + l) * (2 * C) + c;
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      y[o] = hi;
      y[o + C] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
}

__global__ void __launch_bounds__(256)
cl_to_ncl_kernel(const float *__restrict__ x, float *__restrict__ y, int C, int L) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + 8 * i, c = c0 + tx;
    tile[ty + 8 * i][tx] = (c < C && l < L) ? x[((size_t)b * L + l) * C + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, l = l0 + tx;
    if (l < L && c < C) y[((size_t)b * C + c) * L + l] = tile[tx][ty + 8 * i];
  }
}

}  // namespace rave

extern "C" int rave_ncl_to_cl(const float *x, void *y_bf16, float *y_f32, int B, int C, int L, int act,
                              float slope, const float *alpha, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && (y_bf16 || y_f32) && B > 0 && C > 0 && L > 0 && B <= 65535, "ncl_to_cl: bad argument");
  RAVE_CHECK_ARG(act != RAVE_ACT_SNAKE || alpha, "ncl_to_cl: snake needs alpha");
  dim3 grid(ceil_div(L, 32), ceil_div(C, 32), B), block(32, 8);
  ncl_to_cl_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16 *)y_bf16, y_f32, C, L, act, slope,
                                                            alpha);
  RAVE_CHECK_LAUNCH("ncl_to_cl");
  return 0;
}

extern "C" int rave_ncl_to_cl_x3(const float *x, void *y_bf16, int B, int C, int L, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && y_bf16 && B > 0 && C > 0 && L > 0 && B <= 65535, "ncl_to_cl_x3: bad argument");
  dim3 grid(ceil_div(L, 32), ceil_div(C, 32), B), block(32, 8);
  ncl_to_cl_x3_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16 *)y_bf16, C, L);
  RAVE_CHECK_LAUNCH("ncl_to_cl_x3");
  return 0;
}

extern "C" int rave_cl_to_ncl(const float *x_cl, float *y, int B, int C, int L, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x_cl && y && B > 0 && C > 0 && L > 0 && B <= 65535, "cl_to_ncl: bad argument");
  dim3 grid(ceil_div(L, 32), ceil_div(C, 32), B), block(32, 8);
  cl_to_ncl_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x_cl, y, C, L);
  RAVE_CHECK_LAUNCH("cl_to_ncl");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// fused weight preparation for the tensor-core engine:
//   row norms (weight norm)  ->  tap-major bf16 operand layouts for forward AND dgrad in one pass,
// and the inverse on the way back (tap-major fp32 wgrad -> dv, dg).
// ---------------------------------------------------------------------------------------------
namespace rave {

struct TapList {
  int n;
  int tap[32];
};

__global__ void __launch_bounds__(256)
weight_rownorm_kernel(const float *__restrict__ v, float *__restrict__ norm, int R) {
  __shared__ float red[32];
  const int c = blockIdx.x;
  const float *vr = v + (size_t)c * R;
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += blockDim.x) s = fmaf(vr[i], vr[i], s);
  const float n = sqrtf(block_reduce_sum(s, red));
  if (threadIdx.x == 0) norm[c] = n;
}

// v [C0][C1][K] fp32 (+ g[C0], norm[C0] or null) ->
//   outA[t][c0][c1] = bf16(w[c0][c1][tapsA[t]])   dims [nA][C0p][C1p]   (zero in the padded region)
//   outB[t][c1][c0] = bf16(w[c0][c1][tapsB[t]])   dims [nB][C1p][C0p]
// grid (C1p/32, C0p/32), block (32, 8); dynamic smem 32 * (32*K + 1) floats.
__global__ void __launch_bounds__(256)
weight_prep_kernel(const float *__restrict__ v, const float *__restrict__ g, const float *__restrict__ norm,
                   __nv_bfloat16 *__restrict__ outA, TapList tapsA, __nv_bfloat16 *__restrict__ outB,
                   TapList tapsB, int C0, int C1, int K, int C0p, int C1p) {
  extern __shared__ float sw[];   // [32 c0][32*K + 1]
  __shared__ float scale[32];
  const int pitch = 32 * K + 1;
  const int c1t = blockIdx.x * 32, c0t = blockIdx.y * 32;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  if (tid < 32) {
    const int c0 = c0t + tid;
    scale[tid] = (c0 < C0) ? (g ? g[c0] / norm[c0] : 1.f) : 0.f;
  }
  // load: for each of the 32 rows, the contiguous run of 32*K floats starting at (c0, c1t, 0)
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int c0 = c0t + r;
    for (int i = threadIdx.x; i < 32 * K; i += 32) {
      const int c1 = c1t + i / K;
      sw[r * pitch + i] = (c0 < C0 && c1 < C1) ? v[((size_t)c0 * C1 + c1t) * K + i] : 0.f;
    }
  }
  __syncthreads();
  if (outA) {
    for (int t = 0; t < tapsA.n; ++t) {
      const int k = tapsA.tap[t];
      for (int r = threadIdx.y; r < 32; r += 8) {
        const int c0 = c0t + r, c1 = c1t + threadIdx.x;
        if (c0 < C0p && c1 < C1p)
          outA[((size_t)t * C0p + c0) * C1p + c1] = __float2bfloat16_rn(sw[r * pitch + threadIdx.x * K + k] * scale[r]);
      }
    }
  }
  if (outB) {
    for (int t = 0; t < tapsB.n; ++t) {
      const int k = tapsB.tap[t];
      for (int r = threadIdx.y; r < 32; r += 8) {      // r indexes c1 here, threadIdx.x indexes c0
        const int c1 = c1t + r, c0 = c0t + threadIdx.x;
        if (c0 < C0p && c1 < C1p)
          outB[((size_t)t * C1p + c1) * C0p + c0] =
              __float2bfloat16_rn(sw[threadIdx.x * pitch + r * K + k] * scale[threadIdx.x]);
      }
    }
  }
}

// dwt [K][C0p][C1p] fp32 (tap-major wgrad) -> dv [C0][C1][K], dg [C0]   (g == null: dv = dw)
// dwt holds `splits` partial sums ([splits][K][C0p][C1p]); they are combined here in a fixed order
// (deterministic), the combined dw row is staged in dv and then corrected in place.
__global__ void __launch_bounds__(256)
weight_norm_bwd_tapmajor_kernel(const float *__restrict__ dwt, const float *__restrict__ v,
                                const float *__restrict__ g, const float *__restrict__ norm,
                                float *__restrict__ dv, float *__restrict__ dg, int C1, int K, int C0p, int C1p,
                                int splits) {
  __shared__ float red[32];
  const int c0 = blockIdx.x;
  const int R = C1 * K;
  const float *vr = v + (size_t)c0 * R;
  float *dr = dv + (size_t)c0 * R;
  const size_t split_stride = (size_t)K * C0p * C1p;
  float s = 0.f;
  // iterate (k, c1) with c1 fastest: consecutive threads read consecutive addresses of every partial
  for (int j = threadIdx.x; j < R; j += blockDim.x) {
    const int k = j / C1, c1 = j - k * C1;
    const int i = c1 * K + k;                       // index inside the parameter row
    const float *src = dwt + ((size_t)k * C0p + c0) * C1p + c1;
    float dw = 0.f;
    for (int sp = 0; sp < splits; ++sp) dw += src[sp * split_stride];
    dr[i] = dw;
    s = fmaf(dw, vr[i], s);
  }
  if (!g) return;
  const float dot = block_reduce_sum(s, red);   // (also orders the dr writes before the re-reads below)
  const float n = norm[c0];
  const float gn = g[c0] / n;
  const float coef = dot / (n * n);
  for (int i = threadIdx.x; i < R; i += blockDim.x) dr[i] = gn * (dr[i] - vr[i] * coef);
  if (threadIdx.x == 0) dg[c0] = dot / n;
}

}  // namespace rave

extern "C" int rave_weight_prep_tc(const float *v, const float *g, float *norm, void *outA, const int *tapsA,
                                   int nA, void *outB, const int *tapsB, int nB, int C0, int C1, int K, int C0p,
                                   int C1p, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(v && (outA || outB) && C0 > 0 && C1 > 0 && K > 0 && K <= 32, "weight_prep: bad argument");
  RAVE_CHECK_ARG(nA <= 32 && nB <= 32 && C0p >= C0 && C1p >= C1, "weight_prep: bad tap list / padding");
  RAVE_CHECK_ARG(!g || norm, "weight_prep: weight norm needs a norm buffer");
  cudaStream_t s = (cudaStream_t)stream;
  if (g) {
    weight_rownorm_kernel<<<C0, 256, 0, s>>>(v, norm, C1 * K);
    RAVE_CHECK_LAUNCH("weight_rownorm");
  }
  TapList ta, tb;
  ta.n = outA ? nA : 0;
  tb.n = outB ? nB : 0;
  for (int i = 0; i < ta.n; ++i) ta.tap[i] = tapsA[i];
  for (int i = 0; i < tb.n; ++i) tb.tap[i] = tapsB[i];
  const int smem = 32 * (32 * K + 1) * sizeof(float);
  static int attr_bytes = 0;
  if (smem > 48 * 1024 && smem > attr_bytes) {
    cudaFuncSetAttribute(weight_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * (32 * 32 + 1) * 4);
    attr_bytes = 32 * (32 * 32 + 1) * 4;
  }
  dim3 grid(ceil_div(C1p, 32), ceil_div(C0p, 32)), block(32, 8);
  weight_prep_kernel<<<grid, block, smem, s>>>(v, g, norm, (__nv_bfloat16 *)outA, ta, (__nv_bfloat16 *)outB, tb,
                                               C0, C1, K, C0p, C1p);
  RAVE_CHECK_LAUNCH("weight_prep");
  return 0;
}

extern "C" int rave_weight_norm_bwd_tapmajor(const float *dwt, const float *v, const float *g, const float *norm,
                                             float *dv, float *dg, int C0, int C1, int K, int C0p, int C1p,
                                             int splits, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dwt && v && dv && C0 > 0 && C1 > 0 && K > 0, "weight_norm_bwd_tapmajor: bad argument");
  RAVE_CHECK_ARG(!g || (norm && dg), "weight_norm_bwd_tapmajor: weight norm needs norm and dg");
  RAVE_CHECK_ARG(splits >= 1, "weight_norm_bwd_tapmajor: splits must be >= 1");
  weight_norm_bwd_tapmajor_kernel<<<C0, 256, 0, (cudaStream_t)stream>>>(dwt, v, g, norm, dv, dg, C1, K, C0p, C1p,
                                                                       splits);
  RAVE_CHECK_LAUNCH("weight_norm_bwd_tapmajor");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// multi-tensor variants: ONE launch prepares (or back-propagates through the weight norm of) every
// layer of a chain instead of one launch per layer of these tiny kernels; the descriptor table travels by value in the kernel
// parameters (<= 64 layers per launch).
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int MT_MAX = 64;

struct MtLayer {
  const float *v, *g;
  float *norm;
  __nv_bfloat16 *outA, *outB;
  const float *dwt;     // backward only
  float *dv, *dg;       // backward only
  int C0, C1, K, C0p, C1p, nA, nB, splits;
  int wide, J;          // backward with a phase-wide gradient buffer [S][J][C0p][wide*C1p]: tap k lives in slot
                        // tapsA[k] = j*wide + p (0 / 0: plain [S][K][C0p][C1p])
  int row_begin;        // prefix sum of C0 (row-parallel kernels)
  int tile_begin;       // prefix sum of tiles (prep kernel)
  unsigned char tapsA[32], tapsB[32];
};

struct MtTable {
  int n;
  int total_rows, total_tiles, maxK;
  int x3;               // split-operand layouts: out[2][taps][..][..] -- all hi slabs, then all lo slabs
  MtLayer L[MT_MAX];
};

__device__ __forceinline__ int mt_find_row(const MtTable &t, int row) {
  int i = 0;
  while (i + 1 < t.n && t.L[i + 1].row_begin <= row) ++i;
  return i;
}
__device__ __forceinline__ int mt_find_tile(const MtTable &t, int tile) {
  int i = 0;
  while (i + 1 < t.n && t.L[i + 1].tile_begin <= tile) ++i;
  return i;
}

__global__ void __launch_bounds__(256) mt_rownorm_kernel(const __grid_constant__ MtTable t) {
  __shared__ float red[32];
  const int li = mt_find_row(t, blockIdx.x);
  const MtLayer &L = t.L[li];
  if (!L.g) return;
  const int c = blockIdx.x - L.row_begin;
  const int R = L.C1 * L.K;
  const float *vr = L.v + (size_t)c * R;
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += blockDim.x) s = fmaf(vr[i], vr[i], s);
  const float n = sqrtf(block_reduce_sum(s, red));
  if (threadIdx.x == 0) L.norm[c] = n;
}

__global__ void __launch_bounds__(256) mt_prep_kernel(const __grid_constant__ MtTable t) {
  extern __shared__ float sw[];   // [32 c0][32*K + 1]
  __shared__ float scale[32];
  const int li = mt_find_tile(t, blockIdx.x);
  const MtLayer &L = t.L[li];
  const int K = L.K, C0 = L.C0, C1 = L.C1, C0p = L.C0p, C1p = L.C1p;
  const int tiles_x = (C1p + 31) / 32;
  const int tile = blockIdx.x - L.tile_begin;
  const int c1t = (tile % tiles_x) * 32, c0t = (tile / tiles_x) * 32;
  const int pitch = 32 * K + 1;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (threadIdx.x < 32) {
    const int c0 = c0t + threadIdx.x;
    scale[threadIdx.x] = (c0 < C0) ? (L.g ? L.g[c0] / L.norm[c0] : 1.f) : 0.f;
  }
  for (int r = ty; r < 32; r += 8) {
    const int c0 = c0t + r;
    for (int i = tx; i < 32 * K; i += 32) {
      const int c1 = c1t + i / K;
      sw[r * pitch + i] = (c0 < C0 && c1 < C1) ? L.v[((size_t)c0 * C1 + c1t) * K + i] : 0.f;
    }
  }
  __syncthreads();
  if (L.outA) {
    for (int a = 0; a < L.nA; ++a) {
      const int k = L.tapsA[a];
      for (int r = ty; r < 32; r += 8) {
        const int c0 = c0t + r, c1 = c1t + tx;
        if (c0 < C0p && c1 < C1p) {
          const float w = k == 255 ? 0.f : sw[r * pitch + tx * K + k] * scale[r];             // tap -1: zero slab
          const __nv_bfloat16 hi = __float2bfloat16_rn(w);
          if (t.x3) {
            L.outA[((size_t)a * C0p + c0) * C1p + c1] = hi;
            L.outA[((size_t)(L.nA + a) * C0p + c0) * C1p + c1] = __float2bfloat16_rn(w - __bfloat162float(hi));
          } else {
            L.outA[((size_t)a * C0p + c0) * C1p + c1] = hi;
          }
        }
      }
    }
  }
  if (L.outB) {
    for (int b = 0; b < L.nB; ++b) {
      const int k = L.tapsB[b];
      for (int r = ty; r < 32; r += 8) {
        const int c1 = c1t + r, c0 = c0t + tx;
        if (c0 < C0p && c1 < C1p) {
          const float w = k == 255 ? 0.f : sw[tx * pitch + r * K + k] * scale[tx];
          const __nv_bfloat16 hi = __float2bfloat16_rn(w);
          if (t.x3) {
            L.outB[((size_t)b * C1p + c1) * C0p + c0] = hi;
            L.outB[((size_t)(L.nB + b) * C1p + c1) * C0p + c0] = __float2bfloat16_rn(w - __bfloat162float(hi));
          } else {
            L.outB[((size_t)b * C1p + c1) * C0p + c0] = hi;
          }
        }
      }
    }
  }
}

// Shared-memory variant (every row whose tile fits in 96 KB): the split-K partials are read coalesced along c1 and transposed
// into the parameter's own (c1, k) order in SHARED memory, so that v is read and dv written with unit stride, once.  The
// global-memory version below walks v / dv with stride K (K = 15: 60 sectors per warp access for 128 useful bytes) and
// writes dv twice: 0.84 ms of a D-step at ~0.65 TB/s.  Index padding i + i/32 keeps the transposing store conflict-free
// for K = 4, 8, 16 as well as for the odd kernel sizes.
__device__ __forceinline__ int wn_pad(int i) { return i + (i >> 5); }

__global__ void __launch_bounds__(1024) mt_wn_bwd_smem_kernel(const __grid_constant__ MtTable t) {
  extern __shared__ float sh[];
  __shared__ float red[32];
  const int li = mt_find_row(t, blockIdx.x);
  const MtLayer &L = t.L[li];
  if (!L.dwt) return;
  const int c0 = blockIdx.x - L.row_begin;
  const int C1 = L.C1, K = L.K, C0p = L.C0p, C1p = L.C1p;
  const int R = C1 * K;
  const float *vr = L.v + (size_t)c0 * R;
  float *dr = L.dv + (size_t)c0 * R;
  const int wide = L.wide > 1 ? L.wide : 1;
  const size_t split_stride = (size_t)(L.wide > 1 ? L.J : K) * C0p * C1p * wide;
  // four row elements per thread and pass: with 1-2 split-K slices (the large layers) a thread otherwise has a single
  // load in flight and the kernel runs at DRAM latency, not bandwidth
  const int bd = blockDim.x;
  for (int j0 = threadIdx.x; j0 < R; j0 += 4 * bd) {
    const float *src[4];
    int dst[4];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = min(j0 + u * bd, R - 1);                  // (clamped lanes recompute element R-1: same value)
      const int k = j / C1, c1 = j - k * C1;
      const int slot = L.wide > 1 ? (int)L.tapsA[k] : k;
      src[u] = L.dwt + ((size_t)(slot / wide) * C0p + c0) * ((size_t)C1p * wide) + (size_t)(slot % wide) * C1p + c1;
      dst[u] = wn_pad(c1 * K + k);
    }
    for (int sp = 0; sp < L.splits; ++sp) {
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] += __ldg(src[u] + (size_t)sp * split_stride);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (j0 + u * bd < R) sh[dst[u]] = acc[u];
  }
  __syncthreads();
  if (!L.g) {
    for (int i = threadIdx.x; i < R; i += blockDim.x) dr[i] = sh[wn_pad(i)];
    return;
  }
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += blockDim.x) s = fmaf(sh[wn_pad(i)], vr[i], s);
  const float dot = block_reduce_sum(s, red);
  const float n = L.norm[c0];
  const float gn = L.g[c0] / n;
  const float coef = dot / (n * n);
  for (int i = threadIdx.x; i < R; i += blockDim.x) dr[i] = gn * (sh[wn_pad(i)] - vr[i] * coef);
  if (threadIdx.x == 0) L.dg[c0] = dot / n;
}

// Global-memory variant, only for rows whose shared-memory tile would exceed 96 KB (C1 * K above ~23.8 k weights).
__global__ void __launch_bounds__(1024) mt_wn_bwd_kernel(const __grid_constant__ MtTable t) {
  __shared__ float red[32];
  const int li = mt_find_row(t, blockIdx.x);
  const MtLayer &L = t.L[li];
  if (!L.dwt) return;
  const int c0 = blockIdx.x - L.row_begin;
  const int C1 = L.C1, K = L.K, C0p = L.C0p, C1p = L.C1p;
  const int R = C1 * K;
  const float *vr = L.v + (size_t)c0 * R;
  float *dr = L.dv + (size_t)c0 * R;
  const int wide = L.wide > 1 ? L.wide : 1;
  const size_t split_stride = (size_t)(L.wide > 1 ? L.J : K) * C0p * C1p * wide;
  float s = 0.f;
  for (int j = threadIdx.x; j < R; j += blockDim.x) {
    const int k = j / C1, c1 = j - k * C1;
    const int i = c1 * K + k;
    const int slot = L.wide > 1 ? (int)L.tapsA[k] : k;
    const float *src = L.dwt + ((size_t)(slot / wide) * C0p + c0) * ((size_t)C1p * wide) + (size_t)(slot % wide) * C1p + c1;
    // split-K partials: 8 independent loads in flight per thread (the sum was a chain of dependent L2 round trips)
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int sp = 0;
    for (; sp + 8 <= L.splits; sp += 8) {
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] += __ldg(src + (size_t)(sp + u) * split_stride);
    }
    for (; sp < L.splits; ++sp) acc[sp & 7] += __ldg(src + (size_t)sp * split_stride);
    const float dw = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
    dr[i] = dw;
    s = fmaf(dw, vr[i], s);
  }
  if (!L.g) return;
  const float dot = block_reduce_sum(s, red);
  const float n = L.norm[c0];
  const float gn = L.g[c0] / n;
  const float coef = dot / (n * n);
  for (int i = threadIdx.x; i < R; i += blockDim.x) dr[i] = gn * (dr[i] - vr[i] * coef);
  if (threadIdx.x == 0) L.dg[c0] = dot / n;
}

}  // namespace rave

// ---------------------------------------------------------------------------------------------
// Snake on the engine's channel-last bf16 streams (v3 chains on the wgmma kernels): the producing conv writes the
// pre-activation h as bf16, these kernels turn it into the operand a = h + sin^2(alpha h) / (alpha + 1e-9) of the next
// conv (rave/blocks.py:852-860; alpha per channel) and back: g_h = g_a (1 + alpha sin(2 alpha h) / (alpha + 1e-9)) + add,
// dalpha[c] += sum_rows g_a (h sin(2 alpha h) / (alpha+eps) - sin^2(alpha h) / (alpha+eps)^2).  Rows = B * pitch (slack
// rows are zero on both sides: snake(0) = 0).
// ---------------------------------------------------------------------------------------------
namespace rave {

__global__ void __launch_bounds__(256)
snake_cl_fwd_kernel(const __nv_bfloat16 *__restrict__ h, const float *__restrict__ alpha, __nv_bfloat16 *__restrict__ a,
                    long n_vec, int cv) {
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n_vec; i += (long)gridDim.x * 256) {
    const int c0 = (int)(i % cv) * 8;
    const uint4 q = *reinterpret_cast<const uint4 *>(h + i * 8);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = __uint_as_float(w[j] << 16), x1 = __uint_as_float(w[j] & 0xFFFF0000u);
      const float a0 = __ldg(alpha + c0 + 2 * j), a1 = __ldg(alpha + c0 + 2 * j + 1);
      const float s0 = sinf(a0 * x0), s1 = sinf(a1 * x1);
      const __nv_bfloat162 r = __floats2bfloat162_rn(x0 + s0 * s0 / (a0 + 1e-9f), x1 + s1 * s1 / (a1 + 1e-9f));
      o[j] = *reinterpret_cast<const uint32_t *>(&r);
    }
    *reinterpret_cast<uint4 *>(a + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// grid (ceil(C / 64), row blocks); block = 8 channel vectors x 32 row lanes
__global__ void __launch_bounds__(256)
snake_cl_bwd_kernel(const __nv_bfloat16 *__restrict__ ga, const __nv_bfloat16 *__restrict__ h,
                    const float *__restrict__ alpha, const __nv_bfloat16 *__restrict__ add,
                    __nv_bfloat16 *__restrict__ gh, float *__restrict__ dalpha, long rows, int C, int rows_per_block, const BlockSum bs) {
  __shared__ float red[32][64 + 1];
  const int cvl = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int c0 = blockIdx.x * 64 + cvl * 8;
  const bool live = c0 < C;
  float al[8], ae[8], part[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    al[j] = live ? alpha[c0 + j] : 1.f;
    ae[j] = al[j] + 1e-9f;
    part[j] = 0.f;
  }
  const long r0 = (long)blockIdx.y * rows_per_block;
  const long r1 = min(rows, r0 + rows_per_block);
  if (live) {
    for (long r = r0 + rl; r < r1; r += 32) {
      const size_t o = (size_t)r * C + c0;
      const uint4 qg = *reinterpret_cast<const uint4 *>(ga + o);
      const uint4 qh = *reinterpret_cast<const uint4 *>(h + o);
      uint4 qa = make_uint4(0, 0, 0, 0);
      if (add) qa = *reinterpret_cast<const uint4 *>(add + o);
      const uint32_t wg[4] = {qg.x, qg.y, qg.z, qg.w}, wh[4] = {qh.x, qh.y, qh.z, qh.w}, wa[4] = {qa.x, qa.y, qa.z, qa.w};
      uint32_t out[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float res[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float g = e ? __uint_as_float(wg[j] & 0xFFFF0000u) : __uint_as_float(wg[j] << 16);
          const float x = e ? __uint_as_float(wh[j] & 0xFFFF0000u) : __uint_as_float(wh[j] << 16);
          const float ad = e ? __uint_as_float(wa[j] & 0xFFFF0000u) : __uint_as_float(wa[j] << 16);
          const int k = 2 * j + e;
          const float sn = sinf(al[k] * x), s2 = sinf(2.f * al[k] * x);
          res[e] = g * (1.f + al[k] * s2 / ae[k]) + ad;
          part[k] += g * (x * s2 / ae[k] - sn * sn / (ae[k] * ae[k]));
        }
        const __nv_bfloat162 rr = __floats2bfloat162_rn(res[0], res[1]);
        out[j] = *reinterpret_cast<const uint32_t *>(&rr);
      }
      *reinterpret_cast<uint4 *>(gh + o) = make_uint4(out[0], out[1], out[2], out[3]);
    }
  }
  if (!dalpha) return;                      // uniform over the grid
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][cvl * 8 + j] = part[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += red[r][threadIdx.x];
    block_sum_put(bs, threadIdx.x, t);
  }
  block_sum_finish(bs, dalpha);             // one group of 64 channels per grid column
}

}  // namespace rave

extern "C" int rave_snake_cl_fwd(const void *h_bf16, const float *alpha, void *a_bf16, long rows, int C, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(h_bf16 && alpha && a_bf16 && rows > 0 && C > 0 && C % 8 == 0 &&
                     (((uintptr_t)h_bf16 | (uintptr_t)a_bf16) & 15) == 0, "snake_cl_fwd: bad argument (C %% 8, 16-byte rows)");
  const long n_vec = rows * (C / 8);
  long blocks = (n_vec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  snake_cl_fwd_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)h_bf16, alpha,
                                                                     (__nv_bfloat16 *)a_bf16, n_vec, C / 8);
  RAVE_CHECK_LAUNCH("snake_cl_fwd");
  return 0;
}

// dalpha [C] fp32 must be zeroed by the caller (accumulated across blocks); `add` (bf16, same shape) may be null.
extern "C" int rave_snake_cl_bwd(const void *ga_bf16, const void *h_bf16, const float *alpha, const void *add_bf16,
                                 void *gh_bf16, float *dalpha, long rows, int C, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(ga_bf16 && h_bf16 && alpha && gh_bf16 && rows > 0 && C > 0 && C % 8 == 0 &&
                     (((uintptr_t)ga_bf16 | (uintptr_t)h_bf16 | (uintptr_t)gh_bf16 | (uintptr_t)add_bf16) & 15) == 0,
                 "snake_cl_bwd: bad argument (C %% 8, 16-byte rows)");
  const int gx = (C + 63) / 64;
  long gy = (rows + 255) / 256;                 // >= 256 rows per block
  const long cap = (132L * 8 + gx - 1) / gx;
  if (gy > cap) gy = cap;
  if (gy < 1) gy = 1;
  const int rpb = (int)((rows + gy - 1) / gy);
  BlockSum bs;
  memset(&bs, 0, sizeof(bs));
  if (dalpha) {
    if (int rc = block_sum_begin(&bs, (long)gx * gy, 64, (cudaStream_t)stream, 0)) return rc;
    bs.limit = C;
  }
  snake_cl_bwd_kernel<<<dim3(gx, (unsigned)gy), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)ga_bf16, (const __nv_bfloat16 *)h_bf16, alpha, (const __nv_bfloat16 *)add_bf16,
      (__nv_bfloat16 *)gh_bf16, dalpha, rows, C, rpb, bs);
  if (dalpha) block_sum_end(bs, (cudaStream_t)stream);
  RAVE_CHECK_LAUNCH("snake_cl_bwd");
  return 0;
}

// Host-side description of one layer (plain C struct of the ABI)
static int weight_prep_tc_multi_impl(int n, const rave_wprep_layer *layers, void *stream, int x3) {
  using namespace rave;
  RAVE_CHECK_ARG(n > 0 && n <= MT_MAX && layers, "weight_prep_multi: 1..%d layers per call", MT_MAX);
  MtTable t;
  memset(&t, 0, sizeof(t));
  t.n = n;
  int rows = 0, tiles = 0, maxK = 1;
  bool any_g = false;
  for (int i = 0; i < n; ++i) {
    const rave_wprep_layer &h = layers[i];
    RAVE_CHECK_ARG(h.v && h.C0 > 0 && h.C1 > 0 && h.K > 0 && h.K <= 32 && h.nA <= 32 && h.nB <= 32 &&
                       h.C0p >= h.C0 && h.C1p >= h.C1 && (!h.g || h.norm),
                   "weight_prep_multi: bad layer %d", i);
    MtLayer &L = t.L[i];
    L.v = h.v; L.g = h.g; L.norm = h.norm;
    L.outA = (__nv_bfloat16 *)h.outA; L.outB = (__nv_bfloat16 *)h.outB;
    L.C0 = h.C0; L.C1 = h.C1; L.K = h.K; L.C0p = h.C0p; L.C1p = h.C1p;
    L.nA = h.outA ? h.nA : 0; L.nB = h.outB ? h.nB : 0;
    for (int k = 0; k < L.nA; ++k) L.tapsA[k] = (unsigned char)h.tapsA[k];
    for (int k = 0; k < L.nB; ++k) L.tapsB[k] = (unsigned char)h.tapsB[k];
    L.row_begin = rows; L.tile_begin = tiles;
    rows += h.C0;
    tiles += (L.nA || L.nB) ? ceil_div(h.C0p, 32) * ceil_div(h.C1p, 32) : 0;
    if (h.K > maxK) maxK = h.K;
    any_g = any_g || h.g;
  }
  t.total_rows = rows; t.total_tiles = tiles; t.maxK = maxK;
  t.x3 = x3;
  cudaStream_t s = (cudaStream_t)stream;
  if (any_g) {
    mt_rownorm_kernel<<<rows, 256, 0, s>>>(t);
    RAVE_CHECK_LAUNCH("mt_rownorm");
  }
  if (tiles > 0) {
    const int smem = 32 * (32 * maxK + 1) * sizeof(float);
    static int attr_bytes = 0;
    if (smem > 48 * 1024 && smem > attr_bytes) {
      cudaFuncSetAttribute(mt_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * (32 * 32 + 1) * 4);
      attr_bytes = 32 * (32 * 32 + 1) * 4;
    }
    mt_prep_kernel<<<tiles, 256, smem, s>>>(t);
    RAVE_CHECK_LAUNCH("mt_prep");
  }
  return 0;
}

extern "C" int rave_weight_prep_tc_multi(int n, const rave_wprep_layer *layers, void *stream) {
  return weight_prep_tc_multi_impl(n, layers, stream, 0);
}
// split-operand layouts for rave_conv1d_tc_fwd_x3: outA [2][nA][C0p][C1p], outB [2][nB][C1p][C0p] with part 0 = bf16(w),
// part 1 = bf16(w - part 0)
extern "C" int rave_weight_prep_tc_multi_x3(int n, const rave_wprep_layer *layers, void *stream) {
  return weight_prep_tc_multi_impl(n, layers, stream, 1);
}

extern "C" int rave_weight_norm_bwd_multi(int n, const rave_wprep_layer *layers, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(n > 0 && n <= MT_MAX && layers, "weight_norm_bwd_multi: 1..%d layers per call", MT_MAX);
  MtTable t;
  memset(&t, 0, sizeof(t));
  t.n = n;
  int rows = 0, max_row = 0;
  for (int i = 0; i < n; ++i) {
    const rave_wprep_layer &h = layers[i];
    RAVE_CHECK_ARG(h.v && h.dwt && h.dv && h.C0 > 0 && h.C1 > 0 && h.K > 0 && h.splits >= 1 && (!h.g || (h.norm && h.dg)),
                   "weight_norm_bwd_multi: bad layer %d", i);
    MtLayer &L = t.L[i];
    L.v = h.v; L.g = h.g; L.norm = h.norm; L.dwt = h.dwt; L.dv = h.dv; L.dg = h.dg;
    L.C0 = h.C0; L.C1 = h.C1; L.K = h.K; L.C0p = h.C0p; L.C1p = h.C1p; L.splits = h.splits;
    L.wide = h.nA > 1 ? h.nA : 0;
    L.J = h.nB;
    if (L.wide) {
      RAVE_CHECK_ARG(h.K <= 32 && h.nB >= 1, "weight_norm_bwd_multi: bad phase-wide layer %d", i);
      for (int k = 0; k < h.K; ++k) {
        RAVE_CHECK_ARG(h.tapsA[k] >= 0 && h.tapsA[k] < h.nA * h.nB, "weight_norm_bwd_multi: bad tap slot (layer %d)", i);
        L.tapsA[k] = (unsigned char)h.tapsA[k];
      }
    }
    L.row_begin = rows;
    rows += h.C0;
    if (h.C1 * h.K > max_row) max_row = h.C1 * h.K;
  }
  t.total_rows = rows;
  // 256 threads per row: 1024 measured slower in the step (10.39 vs 9.98 ms)
  constexpr int wn_threads = 256;
  const size_t smem = (size_t)(max_row + (max_row >> 5) + 1) * sizeof(float);
  if (smem <= 96 * 1024) {                               // a row of <= ~23.8 k weights; >= 2 CTAs per SM
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(mt_wn_bwd_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      attr = true;
    }
    mt_wn_bwd_smem_kernel<<<rows, wn_threads, smem, (cudaStream_t)stream>>>(t);
    RAVE_CHECK_LAUNCH("mt_wn_bwd_smem");
    return 0;
  }
  mt_wn_bwd_kernel<<<rows, wn_threads, 0, (cudaStream_t)stream>>>(t);
  RAVE_CHECK_LAUNCH("mt_wn_bwd");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Multi-tensor Adam (torch.optim.Adam semantics without weight decay / amsgrad, rave/model.py:226-236): ONE launch per
// <= ADAM_MAX parameter tensors.  lr and the step counter live in device memory (graph-replayable; the LinearLR
// schedule writes lr in place).  PyTorch's capturable foreach path spends ~25 multi-tensor launches plus one scalar
// division per parameter tensor (120-210 launches per step here).
//   m = lerp(m, g, 1-b1);  v = b2 v + (1-b2) g^2;  p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int ADAM_MAX = 96;
constexpr int ADAM_CHUNK = 256 * 4 * 8;      // elements per block

struct AdamTable {
  int n, total_blocks;
  float *p[ADAM_MAX];
  const float *g[ADAM_MAX];
  float *m[ADAM_MAX], *v[ADAM_MAX];
  int numel[ADAM_MAX], block_begin[ADAM_MAX];
};

__global__ void __launch_bounds__(256)
adam_multi_kernel(const __grid_constant__ AdamTable t, const float *__restrict__ lr, const float *__restrict__ step,
                  float b1, float b2, float eps) {
  int i = 0;
  while (i + 1 < t.n && t.block_begin[i + 1] <= (int)blockIdx.x) ++i;
  const int base = ((int)blockIdx.x - t.block_begin[i]) * ADAM_CHUNK;
  const int n = t.numel[i];
  const float st = step[0];
  const float bc1 = 1.f - powf(b1, st), bc2s = sqrtf(1.f - powf(b2, st));
  const float step_size = lr[0] / bc1;
  float *__restrict__ p = t.p[i];
  const float *__restrict__ g = t.g[i];
  float *__restrict__ m = t.m[i];
  float *__restrict__ v = t.v[i];
  for (int j = base + threadIdx.x; j < min(n, base + ADAM_CHUNK); j += 256) {
    const float gj = g[j];
    const float mj = m[j] + (1.f - b1) * (gj - m[j]);
    const float vj = b2 * v[j] + (1.f - b2) * gj * gj;
    m[j] = mj;
    v[j] = vj;
    p[j] -= step_size * mj / (sqrtf(vj) / bc2s + eps);
  }
}

__global__ void adam_step_inc_kernel(float *step) { step[0] += 1.f; }

}  // namespace rave

extern "C" int rave_adam_multi(int n, float *const *params, const float *const *grads, float *const *exp_avg,
                               float *const *exp_avg_sq, const long *numel, const float *lr, float *step, float beta1,
                               float beta2, float eps, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(n > 0 && params && grads && exp_avg && exp_avg_sq && numel && lr && step, "adam_multi: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  adam_step_inc_kernel<<<1, 1, 0, s>>>(step);         // t <- t + 1 first, as torch.optim.Adam does
  RAVE_CHECK_LAUNCH("adam_step");
  for (int i0 = 0; i0 < n; i0 += ADAM_MAX) {
    AdamTable t;
    memset(&t, 0, sizeof(t));
    t.n = (n - i0 < ADAM_MAX) ? n - i0 : ADAM_MAX;
    int blocks = 0;
    for (int i = 0; i < t.n; ++i) {
      RAVE_CHECK_ARG(params[i0 + i] && grads[i0 + i] && exp_avg[i0 + i] && exp_avg_sq[i0 + i] && numel[i0 + i] > 0 &&
                         numel[i0 + i] < (1L << 31),
                     "adam_multi: bad tensor %d", i0 + i);
      t.p[i] = params[i0 + i]; t.g[i] = grads[i0 + i]; t.m[i] = exp_avg[i0 + i]; t.v[i] = exp_avg_sq[i0 + i];
      t.numel[i] = (int)numel[i0 + i];
      t.block_begin[i] = blocks;
      blocks += (int)((numel[i0 + i] + ADAM_CHUNK - 1) / ADAM_CHUNK);
    }
    t.total_blocks = blocks;
    adam_multi_kernel<<<blocks, 256, 0, s>>>(t, lr, step, beta1, beta2, eps);
    RAVE_CHECK_LAUNCH("adam_multi");
  }
  return 0;
}
