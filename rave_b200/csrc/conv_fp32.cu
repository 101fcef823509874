// fp32 CUDA-core conv1d family: the PARITY path (exact fp32 FMA accumulation) and the fallback
// for the small-channel layers (Cin = 1 / Cout = 1) that are not GEMM shaped.
//
// Reference call sites: cc.Conv1d.forward = F.pad + F.conv1d (cached_conv [EXT], used by
// rave/blocks.py:96-108 DilatedUnit, 538-543 stem, 561-575 down-conv, 579-587 head, 637-692
// generator), nn.ConvTranspose1d (blocks.py:650-657), nn.Conv1d / nn.Conv2d (k,1) in
// rave/discriminator.py:99-111, and the autograd (dgrad / wgrad) of each.
//
// One im2col-free implicit GEMM:  out[m][n] = sum_{k} sum_{c} W(m,c,k) * src(n; c,k),
// n = (batch, position).  128x128 output tile per CTA, 8x8 register micro-tile per thread,
// reduction streamed tap by tap in chunks of 8 source channels through double-buffered shared
// memory.  MODE 0 ("gather") reads src at l*stride + k*dil - pad; MODE 1 ("scatter") is the
// transposed map, reading src at (t + pad - k*dil)/stride where divisible.
#include "common.cuh"

namespace rave {

constexpr int TM = 128, TN = 128, TK = 8;

struct ConvArgs {
  const float *src, *w, *bias, *res, *alpha, *post_x, *post_alpha;
  float *out;
  int B, Cs, Ls, Cm, Lo, K, stride, dil, pad_l;
  long ws_m, ws_c;
  int act, post_act;
  float slope, post_slope;
};

template <int MODE>
__global__ void __launch_bounds__(256, 2) conv_f32_kernel(const ConvArgs a) {
  __shared__ __align__(16) float As[2][TK][TM];
  __shared__ __align__(16) float Bs[2][TK][TN];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long N = (long)a.B * a.Lo;
  const long n_tile = (long)blockIdx.x * TN;
  const int m_tile = blockIdx.y * TM;

  // loader coordinates: this thread always fills column/row (tid % 128), kk = tid/128 + 2 i
  const int lcol = tid & 127;
  const int lk0 = tid >> 7;
  const long ln = n_tile + lcol;
  const bool ln_ok = ln < N;
  const int lb = ln_ok ? (int)(ln / a.Lo) : 0;
  const int ll = ln_ok ? (int)(ln - (long)lb * a.Lo) : 0;
  const int lm = m_tile + lcol;
  const bool lm_ok = lm < a.Cm;
  const float *srcb = a.src + (size_t)lb * a.Cs * a.Ls;

  const int nC = ceil_div(a.Cs, TK);
  const int iters = a.K * nC;

  float ra[4], rb[4];
  auto fetch = [&](int it) {
    const int k = it / nC;
    const int c0 = (it - k * nC) * TK;
    int pos;
    bool pos_ok;
    if (MODE == 0) {
      pos = ll * a.stride + k * a.dil - a.pad_l;
      pos_ok = ln_ok && pos >= 0 && pos < a.Ls;
    } else {
      int q = ll + a.pad_l - k * a.dil;
      pos_ok = ln_ok && q >= 0;
      if (a.stride > 1) {
        pos = q / a.stride;
        pos_ok = pos_ok && (pos * a.stride == q);
      } else {
        pos = q;
      }
      pos_ok = pos_ok && pos < a.Ls;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + lk0 + 2 * i;
      float v = 0.f;
      if (pos_ok && c < a.Cs) {
        v = __ldg(srcb + (size_t)c * a.Ls + pos);
        if (a.act) v = act_apply(v, a.act, a.slope, a.act == RAVE_ACT_SNAKE ? __ldg(a.alpha + c) : 0.f);
      }
      rb[i] = v;
      ra[i] = (lm_ok && c < a.Cs) ? __ldg(a.w + lm * a.ws_m + c * a.ws_c + k) : 0.f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][lk0 + 2 * i][lcol] = ra[i];
      Bs[buf][lk0 + 2 * i][lcol] = rb[i];
    }
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  fetch(0);
  stash(0);
  __syncthreads();
  for (int it = 0; it < iters; ++it) {
    const int buf = it & 1;
    if (it + 1 < iters) fetch(it + 1);
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][kk][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < iters) {
      stash(buf ^ 1);
      __syncthreads();
    }
  }

  // epilogue: out = (acc + bias) * post + res
  const bool vec = (a.Lo & 3) == 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m_tile + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= a.Cm) continue;
    const float bias = a.bias ? __ldg(a.bias + m) : 0.f;
    const float palpha = (a.post_act == RAVE_ACT_SNAKE) ? __ldg(a.post_alpha + m) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long n0 = n_tile + h * 64 + tx * 4;
      if (n0 >= N) continue;
      float v[4] = {acc[i][h * 4 + 0] + bias, acc[i][h * 4 + 1] + bias, acc[i][h * 4 + 2] + bias,
                    acc[i][h * 4 + 3] + bias};
      if (vec) {
        const int b = (int)(n0 / a.Lo);
        const int l = (int)(n0 - (long)b * a.Lo);
        const size_t off = ((size_t)b * a.Cm + m) * a.Lo + l;
        if (a.post_act) {
          const float4 px = *reinterpret_cast<const float4 *>(a.post_x + off);
          v[0] *= act_grad(px.x, a.post_act, a.post_slope, palpha);
          v[1] *= act_grad(px.y, a.post_act, a.post_slope, palpha);
          v[2] *= act_grad(px.z, a.post_act, a.post_slope, palpha);
          v[3] *= act_grad(px.w, a.post_act, a.post_slope, palpha);
        }
        if (a.res) {
          const float4 r = *reinterpret_cast<const float4 *>(a.res + off);
          v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
        }
        *reinterpret_cast<float4 *>(a.out + off) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long n = n0 + j;
          if (n >= N) break;
          const int b = (int)(n / a.Lo);
          const int l = (int)(n - (long)b * a.Lo);
          const size_t off = ((size_t)b * a.Cm + m) * a.Lo + l;
          float o = v[j];
          if (a.post_act) o *= act_grad(a.post_x[off], a.post_act, a.post_slope, palpha);
          if (a.res) o += a.res[off];
          a.out[off] = o;
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// wgrad: dW[a][c][k] = sum_b sum_l actP(P[b][a][l]) * actQ(Q[b][c][l*stride + k*dil - pad])
// 64x64 (a x c) tile per CTA for one tap k and one slice of the (b,l) reduction.
// ----------------------------------------------------------------------------------------------
constexpr int WM = 64, WN = 64, WK = 16;

struct WgradArgs {
  const float *P, *Q, *alpha;
  float *part;  // [splits][Ca][Cc][K]
  int B, Ca, Lp, Cc, Lq, K, stride, dil, pad_l, splits, chunks_per_b;
  int act_p, act_q;
  float slope;
};

__global__ void __launch_bounds__(256) conv_wgrad_f32_kernel(const WgradArgs a) {
  __shared__ __align__(16) float As[2][WK][WM + 4];
  __shared__ __align__(16) float Bs[2][WK][WN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int a_tile = blockIdx.y * WM;
  const int c_tile = blockIdx.x * WN;
  const int k = blockIdx.z % a.K;
  const int split = blockIdx.z / a.K;

  const long total_chunks = (long)a.B * a.chunks_per_b;
  const long per = (total_chunks + a.splits - 1) / a.splits;
  const long ch_begin = (long)split * per;
  long ch_end = ch_begin + per;
  if (ch_end > total_chunks) ch_end = total_chunks;

  // loader: kk = tid % 16 (position within the chunk), rows tid/16 + 16 i
  const int lkk = tid & 15;
  const int lr = tid >> 4;
  float ra[4], rb[4];
  auto fetch = [&](long ch) {
    const int b = (int)(ch / a.chunks_per_b);
    const int l = (int)(ch - (long)b * a.chunks_per_b) * WK + lkk;
    const bool l_ok = l < a.Lp;
    const int pos = l * a.stride + k * a.dil - a.pad_l;
    const bool pos_ok = l_ok && pos >= 0 && pos < a.Lq;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int ca = a_tile + lr + 16 * i;
      float v = 0.f;
      if (l_ok && ca < a.Ca) {
        v = __ldg(a.P + ((size_t)b * a.Ca + ca) * a.Lp + l);
        if (a.act_p) v = act_apply(v, a.act_p, a.slope, a.act_p == RAVE_ACT_SNAKE ? __ldg(a.alpha + ca) : 0.f);
      }
      ra[i] = v;
      const int cc = c_tile + lr + 16 * i;
      float u = 0.f;
      if (pos_ok && cc < a.Cc) {
        u = __ldg(a.Q + ((size_t)b * a.Cc + cc) * a.Lq + pos);
        if (a.act_q) u = act_apply(u, a.act_q, a.slope, a.act_q == RAVE_ACT_SNAKE ? __ldg(a.alpha + cc) : 0.f);
      }
      rb[i] = u;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][lkk][lr + 16 * i] = ra[i];
      Bs[buf][lkk][lr + 16 * i] = rb[i];
    }
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  if (ch_begin < ch_end) {
    fetch(ch_begin);
    stash(0);
    __syncthreads();
    int buf = 0;
    for (long ch = ch_begin; ch < ch_end; ++ch) {
      if (ch + 1 < ch_end) fetch(ch + 1);
#pragma unroll
      for (int kk = 0; kk < WK; ++kk) {
        const float4 av = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 4]);
        const float4 bv = *reinterpret_cast<const float4 *>(&Bs[buf][kk][tx * 4]);
        const float aa[4] = {av.x, av.y, av.z, av.w};
        const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
      }
      if (ch + 1 < ch_end) {
        stash(buf ^ 1);
        __syncthreads();
        buf ^= 1;
      }
    }
  }
  float *part = a.part + (size_t)split * a.Ca * a.Cc * a.K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ca = a_tile + ty * 4 + i;
    if (ca >= a.Ca) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int cc = c_tile + tx * 4 + j;
      if (cc >= a.Cc) continue;
      part[((size_t)ca * a.Cc + cc) * a.K + k] = acc[i][j];
    }
  }
}

__global__ void wgrad_reduce_kernel(const float *__restrict__ part, float *__restrict__ dw, int Ca,
                                    int Cc, int K, int splits, long os_a, long os_c) {
  const long total = (long)Ca * Cc * K;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int sp = 0; sp < splits; ++sp) s += part[(size_t)sp * total + i];
    const int k = (int)(i % K);
    const long ac = i / K;
    const int c = (int)(ac % Cc);
    const int aidx = (int)(ac / Cc);
    dw[aidx * os_a + c * os_c + k] = s;
  }
}

static int wgrad_splits(int B, int Ca, int Cc, int Lp, int K) {
  const long tiles = (long)ceil_div(Ca, WM) * ceil_div(Cc, WN) * K;
  const long chunks = (long)B * ceil_div(Lp, WK);
  long want = (132 * 4 + tiles - 1) / tiles;  // ~4 CTAs per SM in flight
  long max_by_work = chunks / 8 > 0 ? chunks / 8 : 1;
  if (want > max_by_work) want = max_by_work;
  if (want < 1) want = 1;
  if (want > 256) want = 256;
  return (int)want;
}

template <int MODE>
static int launch_conv(const ConvArgs &a, void *stream, const char *name) {
  RAVE_CHECK_ARG(a.src && a.w && a.out, "%s: null pointer", name);
  RAVE_CHECK_ARG(a.B > 0 && a.Cs > 0 && a.Ls > 0 && a.Cm > 0 && a.Lo > 0 && a.K > 0 && a.stride > 0 &&
                     a.dil > 0,
                 "%s: bad shape", name);
  RAVE_CHECK_ARG(a.act != RAVE_ACT_SNAKE || a.alpha, "%s: snake needs alpha", name);
  RAVE_CHECK_ARG(!a.post_act || a.post_x, "%s: post_act needs post_x", name);
  RAVE_CHECK_ARG(a.post_act != RAVE_ACT_SNAKE || a.post_alpha, "%s: snake post needs alpha", name);
  const long N = (long)a.B * a.Lo;
  dim3 grid((unsigned)((N + TN - 1) / TN), ceil_div(a.Cm, TM));
  RAVE_CHECK_ARG(grid.y <= 65535, "%s: too many output channels", name);
  conv_f32_kernel<MODE><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  RAVE_CHECK_LAUNCH(name);
  return 0;
}

}  // namespace rave

#define RAVE_FILL_CONV_ARGS()                                                                    \
  rave::ConvArgs a;                                                                              \
  a.src = src; a.w = w; a.bias = bias; a.res = res; a.alpha = alpha; a.post_x = post_x;          \
  a.post_alpha = post_alpha; a.out = out; a.B = B; a.Cs = Cs; a.Ls = Ls; a.Cm = Cm; a.Lo = Lo;    \
  a.K = K; a.stride = stride; a.dil = dil; a.pad_l = pad_l; a.ws_m = ws_m; a.ws_c = ws_c;         \
  a.act = act; a.post_act = post_act; a.slope = slope; a.post_slope = post_slope;

extern "C" int rave_conv1d_gather_f32(const float *src, const float *w, const float *bias,
                                      const float *res, float *out, int B, int Cs, int Ls, int Cm,
                                      int Lo, int K, int stride, int dil, int pad_l, long ws_m,
                                      long ws_c, int act, float slope, const float *alpha,
                                      int post_act, float post_slope, const float *post_x,
                                      const float *post_alpha, void *stream) {
  RAVE_FILL_CONV_ARGS();
  return rave::launch_conv<0>(a, stream, "conv1d_gather_f32");
}

extern "C" int rave_conv1d_scatter_f32(const float *src, const float *w, const float *bias,
                                       const float *res, float *out, int B, int Cs, int Ls, int Cm,
                                       int Lo, int K, int stride, int dil, int pad_l, long ws_m,
                                       long ws_c, int act, float slope, const float *alpha,
                                       int post_act, float post_slope, const float *post_x,
                                       const float *post_alpha, void *stream) {
  RAVE_FILL_CONV_ARGS();
  return rave::launch_conv<1>(a, stream, "conv1d_scatter_f32");
}

extern "C" size_t rave_conv1d_wgrad_workspace_bytes(int B, int Ca, int Cc, int Lp, int K) {
  return (size_t)rave::wgrad_splits(B, Ca, Cc, Lp, K) * Ca * Cc * K * sizeof(float);
}

extern "C" int rave_conv1d_wgrad_f32(const float *P, const float *Q, float *dw, int B, int Ca, int Lp,
                                     int Cc, int Lq, int K, int stride, int dil, int pad_l, long os_a,
                                     long os_c, int act_p, int act_q, float slope, const float *alpha,
                                     void *workspace, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(P && Q && dw && workspace, "conv1d_wgrad: null pointer");
  RAVE_CHECK_ARG(B > 0 && Ca > 0 && Cc > 0 && Lp > 0 && Lq > 0 && K > 0, "conv1d_wgrad: bad shape");
  RAVE_CHECK_ARG((act_p != RAVE_ACT_SNAKE && act_q != RAVE_ACT_SNAKE) || alpha,
                 "conv1d_wgrad: snake needs alpha");
  WgradArgs a;
  a.P = P; a.Q = Q; a.alpha = alpha; a.part = (float *)workspace;
  a.B = B; a.Ca = Ca; a.Lp = Lp; a.Cc = Cc; a.Lq = Lq; a.K = K; a.stride = stride; a.dil = dil;
  a.pad_l = pad_l; a.splits = wgrad_splits(B, Ca, Cc, Lp, K); a.chunks_per_b = ceil_div(Lp, WK);
  a.act_p = act_p; a.act_q = act_q; a.slope = slope;
  dim3 grid(ceil_div(Cc, WN), ceil_div(Ca, WM), K * a.splits);
  RAVE_CHECK_ARG(grid.y <= 65535 && grid.z <= 65535, "conv1d_wgrad: grid too large");
  conv_wgrad_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  RAVE_CHECK_LAUNCH("conv1d_wgrad_f32");
  const long total = (long)Ca * Cc * K;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  wgrad_reduce_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a.part, dw, Ca, Cc, K, a.splits, os_a,
                                                               os_c);
  RAVE_CHECK_LAUNCH("wgrad_reduce");
  return 0;
}
