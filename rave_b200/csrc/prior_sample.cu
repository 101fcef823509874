// Sampling from the latent prior (rave/prior/model.py: Prior.generate, validation_epoch_end):
//   prior_sample          : T frames of classes in one call, one frame of work per step.  The prior is causal and only the
//                           newest frame changes, so each layer keeps the last (K-1)·dil + 1 inputs of its dilated conv in
//                           a ring, and a step runs the stages below on B <= 64 rows:
//                             embed   pre_net on the last K classes (gather of weight columns) + LeakyReLU -> ring 0
//                             gate    per block: dconv on its ring's K taps, CTA owns gate channels c and C + c, so the
//                                     epilogue applies sigmoid · tanh
//                             rs      per block: rconv + sconv as one pass over g; residual into the next block's ring,
//                                     sconv added into the skip vector (the last block has no rconv)
//                             post    post_net.0 + LeakyReLU
//                             head    post_net.2 of each group d, then the class: teacher-forced from the prefix,
//                                     first argmax, or the inverse CDF of the softmax at an explicit uniform
//                           One frame's launches are captured once into a CUDA graph and replayed T - 1 times; the frame
//                           index lives in the workspace and the head advances it.
//   prior_stream          : the exported model's prior(temp) (scripts/export.py TraceModel): the same frame stages on a
//                           state the caller keeps from call to call; the frame graph is captured once per state and
//                           replayed once per frame, and the head also divides the logits by the row's temperature,
//                           decodes the class and writes the diagonally shifted output.
//   prior_classes_to_latent: QuantizedNormal.decode (dither given), DiagonalShift.inverse and
//                           VariationalPrior.pre_process_latent (noise given) in one pass.
// fp32 CUDA-core arithmetic.  Every dot product is added in one fixed order per output (lane-strided partials, then a
// fixed xor tree), which depends on neither B nor the other rows; no float atomics.
#include <vector>

#include "common.cuh"

namespace rave {
namespace {

constexpr int PS_THREADS = 256;
constexpr int PS_WARPS = PS_THREADS / 32;
constexpr int PS_ROWS = 8;              // weight rows staged per CTA in the gate / rs / post stages
constexpr int PS_GATE = PS_ROWS / 2;    // gate channels per CTA
constexpr int PS_NB = 8;                // input rows per pass of the GEMV stages
constexpr int PS_MAX_B = 64, PS_MAX_K = 8, PS_MAX_R = 1024;
constexpr int PS_HEAD_THREADS = 128;
constexpr size_t PS_MAX_SMEM = 200 * 1024;

enum { MODE_GATE = 0, MODE_RES_SKIP = 1, MODE_POST = 2 };

struct Ctl {
  int step;            // frame consumed by the current step
  unsigned ticket;     // head CTAs done with the current step
  // prior_stream only (zero in prior_sample): the call's first produced frame, its length and its tensors, written by
  // the call's prologue so that the one captured frame graph serves calls of any length
  int base, T;
  const float *uniform, *dither;   // [B][T][D]
  float *out;                      // [B][D][T]
};

// Workspace: control word, class ring [B][K][D], per block the ring of dconv inputs [B][S_l][C] with
// S_l = (K-1)·dil_l + 1 (frame t in slot t mod S_l), g [B][C], skip [B][Sk], p [B][Sk]; 256-byte aligned pieces.
struct Layout {
  size_t cls, ring[64], g, skp, p, total;
  int S[64];
  size_t temp, diag;   // prior_stream only
};

inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

Layout layout(int B, int n_layers, int cycle, int C, int Sk, int K, int D) {
  Layout L{};
  size_t o = 256;
  L.cls = o;
  o += up256((size_t)B * K * D * sizeof(int));
  for (int l = 0; l < n_layers; ++l) {
    L.S[l] = (K - 1) * (1 << (l % cycle)) + 1;
    L.ring[l] = o;
    o += up256((size_t)B * L.S[l] * C * sizeof(float));
  }
  L.g = o;
  o += up256((size_t)B * C * sizeof(float));
  L.skp = o;
  o += up256((size_t)B * Sk * sizeof(float));
  L.p = o;
  o += up256((size_t)B * Sk * sizeof(float));
  L.total = o;
  return L;
}

// prior_stream: the sampler's layout, then the row temperatures temp [B] and the diagonal cache [B][D][D]: the decoded
// value of dim d of produced frame n in slot [b][d][n mod D]
Layout stream_layout(int B, int n_layers, int cycle, int C, int Sk, int K, int D) {
  Layout L = layout(B, n_layers, cycle, C, Sk, K, D);
  L.temp = L.total;
  L.diag = L.temp + up256((size_t)B * sizeof(float));
  L.total = L.diag + up256((size_t)B * D * D * sizeof(float));
  return L;
}

// QuantizedNormal.decode of class k with its dither: clamp(erfinv(2 x - 1) sqrt 2, -4, 4), x = k / R + dither / R
__device__ __forceinline__ float class_to_normal(int k, float dither, float rf) {
  const float x = __fadd_rn(__fdiv_rn((float)k, rf), __fdiv_rn(dither, rf));
  const float y = __fmul_rn(erfinvf(__fsub_rn(__fmul_rn(2.f, x), 1.f)), 1.41421356237309515f);
  return fminf(fmaxf(y, -4.f), 4.f);
}

__device__ __forceinline__ int wrap(int t, int S) {
  const int s = t % S;
  return s < 0 ? s + S : s;
}

__global__ void ps_init_kernel(const int *__restrict__ prefix, int *__restrict__ classes, int *__restrict__ cls_ring,
                               int B, int P, int T, int D, int K) {
  const long i = blockIdx.x * (long)PS_THREADS + threadIdx.x;
  if (i >= (long)B * P * D) return;
  const int d = (int)(i % D), t = (int)((i / D) % P), b = (int)(i / ((long)D * P));
  const int k = prefix[i];
  classes[((size_t)b * T + t) * D + d] = k;
  if (t == 0) cls_ring[(size_t)b * K * D + d] = k;
}

// ring0[b][t mod S0][o] = LeakyReLU(bias[o] + sum_{k: t+k-(K-1) >= 0} w[o][c_d(b, t+k-(K-1))][k]), d = o / (C / D):
// prior_embed_fwd_kernel for the one frame t
__global__ void __launch_bounds__(PS_THREADS)
ps_embed_kernel(const Ctl *__restrict__ ctl, const int *__restrict__ cls_ring, const float *__restrict__ w,
                const float *__restrict__ bias, float *__restrict__ ring0, int S0, int B, int C, int D, int R, int K,
                float slope) {
  const int i = blockIdx.x * PS_THREADS + threadIdx.x;
  if (i >= B * C) return;
  const int o = i % C, b = i / C, d = o / (C / D), t = ctl->step;
  const float *wo = w + (size_t)o * R * K;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) {
    const int s = t + k - (K - 1);
    if (s >= 0) acc += wo[cls_ring[((size_t)b * K + s % K) * D + d] * K + k];
  }
  float v = acc + bias[o];
  v = v > 0.f ? v : v * slope;
  ring0[((size_t)b * S0 + t % S0) * C + o] = v;
}

// The GEMV stages.  A CTA stages PS_ROWS weight rows of length J = Cin·K in shared memory, tap-major ([k][i]), then
// takes the input rows b eight at a time; every output is summed in the same order whatever B is.
//   GATE:     rows q < 4: dconv row c0 + q, rows 4 + q: dconv row C + c0 + q; input taps ring[b][(t - (K-1-k) dil)
//             mod S][i]; out[b][c] = sigmoid(h_c) tanh(h_{C+c})
//   RES_SKIP: rows o < na: rconv row o, rows na <= o < na + nb: sconv row o - na; input g[b][i];
//             next ring[b][t mod Sn][o] = ring[b][t mod S][o] + h_o, skip[b][o - na] (+)= h_o
//   POST:     rows o < na of post_net.0; input skip[b][i]; p[b][o] = LeakyReLU(h_o)
struct RowsArgs {
  const Ctl *ctl;
  const float *wa, *ba, *wb, *bb;
  const float *x;          // GATE: ring [B][Sx][Cin]; otherwise [B][Cin]
  float *out;              // GATE: g; RES_SKIP: next ring; POST: p
  const float *res;        // RES_SKIP: the block's ring (residual input)
  float *skp;
  int B, Cin, K, dil, Sx, Sr, Sn, na, nb, first, mode;
  float slope;
};

__device__ __forceinline__ float warp_sum_xor(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// weight row r of the CTA (nullptr past the end) and its bias
__device__ __forceinline__ const float *row_src(const RowsArgs &a, int r, int J, float *bias, int *o) {
  if (a.mode == MODE_GATE) {
    const int c = blockIdx.x * PS_GATE + r % PS_GATE, h = r / PS_GATE * a.na + c;
    *o = c;
    if (c >= a.na) return nullptr;
    *bias = a.ba[h];
    return a.wa + (size_t)h * J;
  }
  const int row = blockIdx.x * PS_ROWS + r;
  *o = row;
  if (row < a.na) { *bias = a.ba[row]; return a.wa + (size_t)row * J; }
  if (row < a.na + a.nb) { *bias = a.bb[row - a.na]; return a.wb + (size_t)(row - a.na) * J; }
  return nullptr;
}

__global__ void __launch_bounds__(PS_THREADS) ps_rows_kernel(const RowsArgs a) {
  extern __shared__ float sw[];                 // [PS_ROWS][K][Cin]
  const int Cin = a.Cin, K = a.K, J = Cin * K, tid = threadIdx.x;
  const int t = a.ctl->step;
  // stage the rows transposed to [k][i]; four independent loads in flight per thread
  const bool vec = (J & 3) == 0 && ((uintptr_t)a.wa & 15) == 0 && ((uintptr_t)a.wb & 15) == 0;
  const int per = vec ? J / 4 : J, n = PS_ROWS * per;
  for (int base = tid; base < n; base += 4 * PS_THREADS) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = base + u * PS_THREADS, r = e / per, j = e - r * per;
      float bias;
      int o;
      const float *src = e < n ? row_src(a, r, J, &bias, &o) : nullptr;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (src) {
        if (vec) v[u] = __ldg(reinterpret_cast<const float4 *>(src) + j);
        else v[u].x = __ldg(src + j);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = base + u * PS_THREADS, r = e / per, j = e - r * per;
      if (e >= n) break;
      float *dst = sw + (size_t)r * J;
      const float vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!vec && q > 0) break;
        const int jj = vec ? 4 * j + q : j, i = jj / K, k = jj - i * K;
        dst[k * Cin + i] = vv[q];
      }
    }
  }
  __syncthreads();

  // PS_NB input rows per pass; thread tid adds j = tid, tid + 256, ... (tap-major), then a fixed xor tree per warp and
  // the 8 warp partials in warp order
  __shared__ float red[PS_WARPS][PS_NB][PS_ROWS];
  const int warp = tid >> 5, lane = tid & 31;
  for (int b0 = 0; b0 < a.B; b0 += PS_NB) {
    const int nb = min(PS_NB, a.B - b0);
    float acc[PS_NB][PS_ROWS];
#pragma unroll
    for (int q = 0; q < PS_NB; ++q)
#pragma unroll
      for (int r = 0; r < PS_ROWS; ++r) acc[q][r] = 0.f;
    for (int j = tid; j < J; j += PS_THREADS) {
      const int k = j / Cin, i = j - k * Cin;
      const float *xj = a.x + (size_t)wrap(t - (K - 1 - k) * a.dil, a.Sx) * Cin + i;
      float wv[PS_ROWS];
#pragma unroll
      for (int r = 0; r < PS_ROWS; ++r) wv[r] = sw[(size_t)r * J + j];
#pragma unroll
      for (int q = 0; q < PS_NB; ++q)
        if (q < nb) {
          const float xv = xj[(size_t)(b0 + q) * a.Sx * Cin];
#pragma unroll
          for (int r = 0; r < PS_ROWS; ++r) acc[q][r] = fmaf(wv[r], xv, acc[q][r]);
        }
    }
#pragma unroll
    for (int q = 0; q < PS_NB; ++q)
#pragma unroll
      for (int r = 0; r < PS_ROWS; ++r) {
        const float v = warp_sum_xor(acc[q][r]);
        if (lane == 0) red[warp][q][r] = v;
      }
    __syncthreads();
    if (tid < PS_NB * PS_ROWS) {
      const int q = tid / PS_ROWS, r = tid % PS_ROWS, b = b0 + q;
      float bias = 0.f, h = 0.f;
      int o;
      const bool has = row_src(a, r, J, &bias, &o) != nullptr;
      for (int w = 0; w < PS_WARPS; ++w) h += red[w][q][r];
      h += bias;
      if (q < nb && has) {
        if (a.mode == MODE_GATE) {
          if (r < PS_GATE) {
            float bias2 = 0.f, h2 = 0.f;
            int o2;
            row_src(a, r + PS_GATE, J, &bias2, &o2);
            for (int w = 0; w < PS_WARPS; ++w) h2 += red[w][q][r + PS_GATE];
            h2 += bias2;
            const float sg = 1.f / (1.f + expf(-h));
            a.out[(size_t)b * a.na + o] = sg * tanhf(h2);
          }
        } else if (a.mode == MODE_RES_SKIP) {
          if (o < a.na) {
            const float x0 = a.res[((size_t)b * a.Sr + t % a.Sr) * a.na + o];
            a.out[((size_t)b * a.Sn + t % a.Sn) * a.na + o] = x0 + h;
          } else {
            float *sp = a.skp + (size_t)b * a.nb + (o - a.na);
            *sp = a.first ? h : *sp + h;
          }
        } else {
          a.out[(size_t)b * a.na + o] = h > 0.f ? h : h * a.slope;
        }
      }
    }
    __syncthreads();
  }
}

// CTA (d, b): logits l[r] = bias[d R + r] + sum_j w[d R + r][j] p[b][d Cg + j] (j in order), then the class of frame
// t + 1: prefix[b][t + 1][d] while t + 1 < P, else the first argmax, else the inverse CDF: the first r whose running sum
// of softmax probabilities (max subtracted, classes 0..R-1 in order) exceeds u = uniform[b][t + 1][d], or the last r of
// non-zero probability if rounding leaves none.  The last CTA to finish advances the frame index.
// prior_stream (diag non-null): the logits are divided by the row's temperature temp[b] first, the uniform is
// ctl->uniform[b][f][d] with f = t + 1 - ctl->base the frame's index in the call, and the CTA then decodes its class with
// ctl->dither[b][f][d] into diag[b][d][(t + 1) mod D] and writes ctl->out[b][d][f] = diag[b][d][(t + 1 - (D-1-d)) mod D]
// (DiagonalShift.inverse: dim d lags the newest frame by D - 1 - d frames).
__global__ void __launch_bounds__(PS_HEAD_THREADS)
ps_head_kernel(Ctl *__restrict__ ctl, const float *__restrict__ p, const float *__restrict__ w,
               const float *__restrict__ bias, const int *__restrict__ prefix, const float *__restrict__ uniform,
               int *__restrict__ classes, int *__restrict__ cls_ring, float *__restrict__ logits, int Sk, int D, int R,
               int K, int P, int T, int argmax, const float *__restrict__ temp, float *__restrict__ diag) {
  __shared__ float lg[PS_MAX_R];
  const int d = blockIdx.x, b = blockIdx.y, Cg = Sk / D, t = ctl->step;
  const float *pb = p + (size_t)b * Sk + (size_t)d * Cg;
  for (int r = threadIdx.x; r < R; r += PS_HEAD_THREADS) {
    const float *wr = w + ((size_t)d * R + r) * Cg;
    float acc = 0.f;
    for (int j = 0; j < Cg; ++j) acc = fmaf(wr[j], pb[j], acc);
    const float l = acc + bias[d * R + r];
    lg[r] = diag ? __fdiv_rn(l, temp[b]) : l;
    if (logits) logits[(((size_t)b * (T - 1) + t) * D + d) * R + r] = l;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int f = t + 1;
  if (diag) {
    f -= ctl->base;
    T = ctl->T;
    uniform = ctl->uniform;
  }
  int k;
  if (t + 1 < P) {
    k = prefix[((size_t)b * P + t + 1) * D + d];
  } else if (argmax) {
    k = 0;
    for (int r = 1; r < R; ++r)
      if (lg[r] > lg[k]) k = r;
  } else {
    float m = lg[0];
    for (int r = 1; r < R; ++r) m = fmaxf(m, lg[r]);
    float s = 0.f;
    for (int r = 0; r < R; ++r) s += expf(lg[r] - m);
    const float u = uniform[((size_t)b * T + f) * D + d];
    float cum = 0.f;
    int last = 0;
    k = -1;
    for (int r = 0; r < R; ++r) {
      const float pr = expf(lg[r] - m) / s;
      if (pr > 0.f) last = r;
      cum += pr;
      if (cum > u) { k = r; break; }
    }
    if (k < 0) k = last;
  }
  if (diag) {
    float *db = diag + ((size_t)b * D + d) * D;
    db[(t + 1) % D] = class_to_normal(k, ctl->dither[((size_t)b * T + f) * D + d], (float)R);
    ctl->out[((size_t)b * D + d) * T + f] = db[wrap(t + 1 - (D - 1 - d), D)];
  } else {
    classes[((size_t)b * T + t + 1) * D + d] = k;
  }
  cls_ring[((size_t)b * K + (t + 1) % K) * D + d] = k;
  __threadfence();
  if (atomicAdd(&ctl->ticket, 1u) == gridDim.x * gridDim.y - 1) {
    ctl->ticket = 0;
    ctl->step = t + 1;
    __threadfence();
  }
}

// z[b][l][t] = latent_mean[l] + sum_c pca[c][l] y[c],  y[c < D] = clamp(erfinv(2 x - 1) sqrt 2, -4, 4),
// x = k / R + dither / R of class k = classes[b][t + c][d = c] (DiagonalShift.inverse), y[c >= D] = noise[b][c - D][t]
__global__ void __launch_bounds__(PS_THREADS)
ps_latent_kernel(const int *__restrict__ cls, const float *__restrict__ dither, const float *__restrict__ noise,
                 const float *__restrict__ pca, const float *__restrict__ lmean, float *__restrict__ z, int B, int T,
                 int D, int L, int R) {
  const int Tq = T - D + 1;
  const long i = blockIdx.x * (long)PS_THREADS + threadIdx.x;
  if (i >= (long)B * L * Tq) return;
  const int t = (int)(i % Tq), l = (int)((i / Tq) % L), b = (int)(i / ((long)Tq * L));
  const float rf = (float)R;
  float acc = 0.f;
  for (int c = 0; c < L; ++c) {
    float y;
    if (c < D) {
      const size_t e = ((size_t)b * T + t + c) * D + c;
      y = class_to_normal(cls[e], dither[e], rf);
    } else {
      y = noise[((size_t)b * (L - D) + (c - D)) * Tq + t];
    }
    acc = fmaf(pca[(size_t)c * L + l], y, acc);
  }
  z[i] = acc + lmean[l];
}

inline int blocks_of(long n) { return (int)((n + PS_THREADS - 1) / PS_THREADS); }

size_t rows_smem(int Cin, int K) { return (size_t)PS_ROWS * Cin * K * sizeof(float); }

struct Plan {
  const float *const *prm;
  int n_layers, cycle, C, Sk, K, R, D, B, P, T, argmax;
  const int *prefix;
  const float *uniform;
  int *classes;
  float *logits;
  char *work;
  Layout L;
  bool stream = false;     // prior_stream: temperature and diagonal-cache output in the head
};

// one step: frame ctl->step in, frame ctl->step + 1 out
void enqueue_frame(const Plan &q, cudaStream_t s) {
  const Layout &L = q.L;
  Ctl *ctl = reinterpret_cast<Ctl *>(q.work);
  int *cls_ring = reinterpret_cast<int *>(q.work + L.cls);
  float *g = reinterpret_cast<float *>(q.work + L.g), *skp = reinterpret_cast<float *>(q.work + L.skp);
  float *p = reinterpret_cast<float *>(q.work + L.p);
  auto ring = [&](int l) { return reinterpret_cast<float *>(q.work + L.ring[l]); };
  const float *const *prm = q.prm;
  ps_embed_kernel<<<blocks_of((long)q.B * q.C), PS_THREADS, 0, s>>>(ctl, cls_ring, prm[0], prm[1], ring(0), L.S[0],
                                                                    q.B, q.C, q.D, q.R, q.K, 0.2f);
  for (int l = 0; l < q.n_layers; ++l) {
    const float *const *lp = prm + 2 + 6 * l;
    const bool last = l == q.n_layers - 1;
    RowsArgs ga{ctl, lp[0], lp[1], nullptr, nullptr, ring(l), g, nullptr, nullptr,
                q.B, q.C, q.K, 1 << (l % q.cycle), L.S[l], 0, 0, q.C, 0, 0, MODE_GATE, 0.f};
    ps_rows_kernel<<<ceil_div(q.C, PS_GATE), PS_THREADS, rows_smem(q.C, q.K), s>>>(ga);
    const int na = last ? 0 : q.C;
    RowsArgs ra{ctl, lp[2], lp[3], lp[4], lp[5], g, last ? nullptr : ring(l + 1), ring(l), skp,
                q.B, q.C, 1, 1, 1, L.S[l], last ? 1 : L.S[l + 1], na, q.Sk, l == 0, MODE_RES_SKIP, 0.f};
    ps_rows_kernel<<<ceil_div(na + q.Sk, PS_ROWS), PS_THREADS, rows_smem(q.C, 1), s>>>(ra);
  }
  const float *const *pp = prm + 2 + 6 * q.n_layers;
  RowsArgs pa{ctl, pp[0], pp[1], nullptr, nullptr, skp, p, nullptr, nullptr,
              q.B, q.Sk, 1, 1, 1, 0, 0, q.Sk, 0, 0, MODE_POST, 0.2f};
  ps_rows_kernel<<<ceil_div(q.Sk, PS_ROWS), PS_THREADS, rows_smem(q.Sk, 1), s>>>(pa);
  ps_head_kernel<<<dim3(q.D, q.B), PS_HEAD_THREADS, 0, s>>>(ctl, p, pp[2], pp[3], q.prefix, q.uniform, q.classes,
                                                           cls_ring, q.logits, q.Sk, q.D, q.R, q.K, q.P, q.T,
                                                           q.argmax,
                                                           q.stream ? reinterpret_cast<float *>(q.work + L.temp) : nullptr,
                                                           q.stream ? reinterpret_cast<float *>(q.work + L.diag) : nullptr);
}

// prologue of a prior_stream call: temp[b] = softplus(mean_t temp_in[b][0][t]) / ln 2 (beta 1, threshold 20, the mean
// summed in t order), and the call's frame base, length and tensors into the control block
__global__ void ps_prologue_kernel(Ctl *__restrict__ ctl, const float *__restrict__ temp_in, float *__restrict__ temp,
                                   const float *uniform, const float *dither, float *out, int B, int T) {
  const int b = threadIdx.x;
  if (b < B) {
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += temp_in[(size_t)b * T + t];
    const float m = __fdiv_rn(s, (float)T);
    const float sp = m > 20.f ? m : log1pf(expf(m));
    temp[b] = __fdiv_rn(sp, 0.693147180559945309f);
  }
  if (b == 0) {
    ctl->base = ctl->step + 1;
    ctl->T = T;
    ctl->uniform = uniform;
    ctl->dither = dither;
    ctl->out = out;
  }
}

// initial state of a prior_stream: frame 0 is QuantizedNormal.encode(0), class R / 2 in every dim
__global__ void ps_reset_kernel(int *__restrict__ cls_ring, int B, int K, int D, int R) {
  const int i = blockIdx.x * PS_THREADS + threadIdx.x;
  if (i < B * D) cls_ring[(size_t)(i / D) * K * D + i % D] = R / 2;
}

// checks shared by prior_sample and prior_stream_create; sets the stages' shared-memory limit
int check_net(const char *who, const float *const *params, int n_layers, int cycle_size, int res_size, int skp_size,
              int K, int R, int D, int B) {
  RAVE_CHECK_ARG(B >= 1 && B <= PS_MAX_B, "%s: B = %d, want 1 <= B <= %d", who, B, PS_MAX_B);
  RAVE_CHECK_ARG(n_layers >= 1 && n_layers <= 64 && cycle_size >= 1 && cycle_size <= 16,
                 "%s: n_layers %d (1..64), cycle_size %d (1..16)", who, n_layers, cycle_size);
  RAVE_CHECK_ARG(D >= 1 && res_size >= 1 && skp_size >= 1 && res_size % D == 0 && skp_size % D == 0,
                 "%s: D = %d must divide res_size %d and skp_size %d", who, D, res_size, skp_size);
  RAVE_CHECK_ARG(K >= 1 && K <= PS_MAX_K, "%s: kernel_size %d, want 1..%d", who, K, PS_MAX_K);
  RAVE_CHECK_ARG(R >= 1 && R <= PS_MAX_R, "%s: resolution %d, want 1..%d", who, R, PS_MAX_R);
  const size_t smem = rows_smem(res_size, K);
  RAVE_CHECK_ARG(smem <= PS_MAX_SMEM && rows_smem(skp_size, 1) <= PS_MAX_SMEM,
                 "%s: res_size * kernel_size = %d too large", who, res_size * K);
  for (int i = 0; i < 2 + 6 * n_layers + 4; ++i) RAVE_CHECK_ARG(params[i], "%s: parameter %d is null", who, i);
  const size_t smem_max = smem > rows_smem(skp_size, 1) ? smem : rows_smem(skp_size, 1);
  if (cudaFuncSetAttribute(ps_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max) != cudaSuccess) {
    cudaGetLastError();
    set_error("%s: %zu bytes of shared memory refused", who, smem_max);
    return 2;
  }
  return 0;
}

int check_not_capturing(const char *who, cudaStream_t s) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  RAVE_CHECK_ARG(cudaStreamIsCapturing(s, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone,
                 "%s: the stream is being captured; the call replays its own CUDA graph once per frame, "
                 "so it cannot run inside a stream capture", who);
  return 0;
}

// One frame's launches captured on a private stream (measured faster than enqueueing the stages frame by frame,
// DESIGN.md §5.8b) and instantiated.
cudaError_t capture_frame(const Plan &q, cudaGraphExec_t *exec) {
  cudaStream_t cs = nullptr;
  cudaGraph_t graph = nullptr;
  *exec = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
  if (e == cudaSuccess) {
    enqueue_frame(q, cs);
    const cudaError_t el = cudaGetLastError();
    e = cudaStreamEndCapture(cs, &graph);
    if (e == cudaSuccess) e = el;
  }
  if (e == cudaSuccess) e = cudaGraphInstantiate(exec, graph, 0);
  if (graph) cudaGraphDestroy(graph);
  if (cs) cudaStreamDestroy(cs);
  return e;
}

// a prior_stream: the plan of its frame graph (parameter pointers copied) and the graph
struct PriorStream {
  std::vector<const float *> prm;
  Plan q;
  cudaGraphExec_t exec;
};

}  // namespace
}  // namespace rave

extern "C" long rave_prior_sample_workspace_bytes(int B, int n_layers, int cycle_size, int res_size, int skp_size,
                                                  int K, int D) {
  if (B < 1 || n_layers < 1 || n_layers > 64 || cycle_size < 1 || cycle_size > 16 || res_size < 1 || skp_size < 1 ||
      K < 1 || D < 1)
    return -1;
  return (long)rave::layout(B, n_layers, cycle_size, res_size, skp_size, K, D).total;
}

extern "C" int rave_prior_sample(const float *const *params, int n_layers, int cycle_size, int res_size, int skp_size,
                                 int K, int R, int D, const int *prefix, int P, const float *uniform, int T, int B,
                                 int argmax, int *classes, float *logits, void *work, long work_bytes, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(params && prefix && classes && work && (argmax || uniform), "prior_sample: null pointer");
  RAVE_CHECK_ARG(P >= 1 && P <= T, "prior_sample: prefix of %d frames for %d frames, want 1 <= P <= T", P, T);
  if (const int rc = check_net("prior_sample", params, n_layers, cycle_size, res_size, skp_size, K, R, D, B)) return rc;
  const Layout L = layout(B, n_layers, cycle_size, res_size, skp_size, K, D);
  RAVE_CHECK_ARG(work_bytes >= (long)L.total, "prior_sample: workspace of %ld bytes, need %zu", work_bytes, L.total);
  const cudaStream_t s = (cudaStream_t)stream;
  if (const int rc = check_not_capturing("prior_sample", s)) return rc;

  char *w = static_cast<char *>(work);
  cudaMemsetAsync(w, 0, L.total, s);
  ps_init_kernel<<<blocks_of((long)B * P * D), PS_THREADS, 0, s>>>(prefix, classes, reinterpret_cast<int *>(w + L.cls),
                                                                   B, P, T, D, K);
  RAVE_CHECK_LAUNCH("prior_sample");
  if (T == 1) return 0;
  const Plan q{params, n_layers, cycle_size, res_size, skp_size, K, R, D, B, P, T, argmax != 0, prefix, uniform,
               classes, logits, w, L};
  cudaGraphExec_t exec = nullptr;
  cudaError_t e = capture_frame(q, &exec);
  for (int i = 0; e == cudaSuccess && i < T - 1; ++i) e = cudaGraphLaunch(exec, s);
  if (exec) cudaGraphExecDestroy(exec);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("prior_sample: frame graph failed: %s", cudaGetErrorString(e));
    return 2;
  }
  count_launch(T - 1);
  return 0;
}

extern "C" long rave_prior_stream_workspace_bytes(int B, int n_layers, int cycle_size, int res_size, int skp_size,
                                                  int K, int D) {
  if (B < 1 || n_layers < 1 || n_layers > 64 || cycle_size < 1 || cycle_size > 16 || res_size < 1 || skp_size < 1 ||
      K < 1 || D < 1)
    return -1;
  return (long)rave::stream_layout(B, n_layers, cycle_size, res_size, skp_size, K, D).total;
}

extern "C" int rave_prior_stream_create(const float *const *params, int n_layers, int cycle_size, int res_size,
                                        int skp_size, int K, int R, int D, int B, void *work, long work_bytes,
                                        void **state) {
  using namespace rave;
  RAVE_CHECK_ARG(params && work && state, "prior_stream_create: null pointer");
  if (const int rc = check_net("prior_stream_create", params, n_layers, cycle_size, res_size, skp_size, K, R, D, B))
    return rc;
  const Layout L = stream_layout(B, n_layers, cycle_size, res_size, skp_size, K, D);
  RAVE_CHECK_ARG(work_bytes >= (long)L.total, "prior_stream_create: workspace of %ld bytes, need %zu", work_bytes,
                 L.total);
  auto *ps = new PriorStream;
  ps->prm.assign(params, params + 2 + 6 * n_layers + 4);
  ps->q = Plan{ps->prm.data(), n_layers, cycle_size, res_size, skp_size, K, R, D, B, 0, 0, 0, nullptr, nullptr,
               nullptr, nullptr, static_cast<char *>(work), L, true};
  const cudaError_t e = capture_frame(ps->q, &ps->exec);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (ps->exec) cudaGraphExecDestroy(ps->exec);
    delete ps;
    set_error("prior_stream_create: frame graph capture failed: %s", cudaGetErrorString(e));
    return 2;
  }
  *state = ps;
  return 0;
}

extern "C" int rave_prior_stream_reset(void *state, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(state, "prior_stream_reset: null state");
  const Plan &q = static_cast<PriorStream *>(state)->q;
  const cudaStream_t s = (cudaStream_t)stream;
  cudaMemsetAsync(q.work, 0, q.L.total, s);
  ps_reset_kernel<<<blocks_of((long)q.B * q.D), PS_THREADS, 0, s>>>(reinterpret_cast<int *>(q.work + q.L.cls),
                                                                   q.B, q.K, q.D, q.R);
  RAVE_CHECK_LAUNCH("prior_stream_reset");
  return 0;
}

extern "C" int rave_prior_stream(void *state, const float *temp, const float *uniform, const float *dither, float *out,
                                 int T, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(state && temp && uniform && dither && out, "prior_stream: null pointer");
  RAVE_CHECK_ARG(T >= 1, "prior_stream: T = %d frames, want T >= 1", T);
  const cudaStream_t s = (cudaStream_t)stream;
  if (const int rc = check_not_capturing("prior_stream", s)) return rc;
  const PriorStream *ps = static_cast<PriorStream *>(state);
  const Plan &q = ps->q;
  ps_prologue_kernel<<<1, PS_MAX_B, 0, s>>>(reinterpret_cast<Ctl *>(q.work), temp,
                                             reinterpret_cast<float *>(q.work + q.L.temp), uniform, dither, out, q.B, T);
  RAVE_CHECK_LAUNCH("prior_stream");
  cudaError_t e = cudaSuccess;
  for (int i = 0; e == cudaSuccess && i < T; ++i) e = cudaGraphLaunch(ps->exec, s);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("prior_stream: frame graph failed: %s", cudaGetErrorString(e));
    return 2;
  }
  count_launch(T);
  return 0;
}

extern "C" int rave_prior_stream_destroy(void *state) {
  auto *ps = static_cast<rave::PriorStream *>(state);
  if (ps) {
    cudaGraphExecDestroy(ps->exec);
    delete ps;
  }
  return 0;
}

extern "C" int rave_prior_classes_to_latent(const int *classes, const float *dither, const float *noise,
                                            const float *latent_pca, const float *latent_mean, float *z, int B, int T,
                                            int D, int L, int R, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(classes && dither && latent_pca && latent_mean && z && (noise || L == D),
                 "prior_classes_to_latent: null pointer");
  RAVE_CHECK_ARG(B >= 1 && D >= 1 && L >= D && T >= D && R >= 1,
                 "prior_classes_to_latent: bad shape (B %d, T %d, D %d, L %d, R %d)", B, T, D, L, R);
  const long n = (long)B * L * (T - D + 1);
  ps_latent_kernel<<<blocks_of(n), PS_THREADS, 0, (cudaStream_t)stream>>>(classes, dither, noise, latent_pca,
                                                                         latent_mean, z, B, T, D, L, R);
  RAVE_CHECK_LAUNCH("prior_classes_to_latent");
  return 0;
}
