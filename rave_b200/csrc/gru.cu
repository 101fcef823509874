// Multi-layer GRU of the hybrid generator head (rave/blocks.py:295-319: nn.GRU(H, H, num_layers, batch_first=True),
// PyTorch's gate order r, z, n):
//     r = sigmoid(gi_r + W_hr h + b_hr)      z = sigmoid(gi_z + W_hz h + b_hz)
//     hn = W_hn h + b_hn                     n = tanh(gi_n + r * hn)             h' = (1 - z) n + z h
// with gi = W_ih x_t + b_ih computed for every t by one GEMM before the recurrence (rave_gemm_f32).
//
// rave_gru_fwd / rave_gru_bwd run the whole time loop of one layer in ONE persistent launch: each CTA owns GRU_ROWS
// batch rows (rows are independent) and keeps W_hh (3H x H fp32 = 192 KB at H = 128) in shared memory for all T steps.
// Everything is fp32 and every sum has a fixed order: two runs are bit-identical.
//
// rave_gemm_f32: C = A B (+ bias) over general strides, plus optionally the row sums of A (bias gradients), with a
// fixed-order split-K: the input projection, dx and the weight / bias gradients of the GRU are GEMMs over B*T rows.
#include "common.cuh"

namespace rave {

constexpr int GRU_H = 128;
constexpr int GRU_G = 3 * GRU_H;        // gate rows; one thread per gate row
constexpr int GRU_ROWS = 2;             // batch rows per CTA

__device__ __forceinline__ float gru_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// smem: W4[k4][j] = W_hh[j][4k4 .. 4k4+3] (float4, conflict-free per warp), h[ROWS][H], gh[ROWS][3H]
__global__ void __launch_bounds__(GRU_G, 1)
gru_fwd_kernel(const float *__restrict__ gi, const float *__restrict__ w_hh, const float *__restrict__ b_hh,
               float *__restrict__ h_out, float *__restrict__ save, int B, int T) {
  extern __shared__ float4 smem4[];
  float4 *W4 = smem4;                                            // [H/4][3H]
  float *hs = reinterpret_cast<float *>(W4 + (GRU_H / 4) * GRU_G);  // [ROWS][H]
  float *ghs = hs + GRU_ROWS * GRU_H;                              // [ROWS][3H]
  const int tid = threadIdx.x;
  const int b0 = blockIdx.x * GRU_ROWS;
  for (int idx = tid; idx < (GRU_H / 4) * GRU_G; idx += GRU_G) {
    const int k4 = idx / GRU_G, j = idx % GRU_G;
    W4[idx] = *reinterpret_cast<const float4 *>(w_hh + (size_t)j * GRU_H + 4 * k4);
  }
  for (int idx = tid; idx < GRU_ROWS * GRU_H; idx += GRU_G) hs[idx] = 0.f;     // h0 = 0 (nn.GRU without hx)
  const float bj = b_hh[tid];
  // gate phase mapping: thread -> (row, hidden index)
  const int gb = tid / GRU_H, gi_ = tid % GRU_H;
  const bool gate_thread = tid < GRU_ROWS * GRU_H && b0 + gb < B;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    float acc[GRU_ROWS];
#pragma unroll
    for (int b = 0; b < GRU_ROWS; ++b) acc[b] = bj;
#pragma unroll 4
    for (int k4 = 0; k4 < GRU_H / 4; ++k4) {
      const float4 w = W4[k4 * GRU_G + tid];
#pragma unroll
      for (int b = 0; b < GRU_ROWS; ++b) {
        const float4 hv = reinterpret_cast<const float4 *>(hs + b * GRU_H)[k4];
        acc[b] = fmaf(w.x, hv.x, acc[b]);
        acc[b] = fmaf(w.y, hv.y, acc[b]);
        acc[b] = fmaf(w.z, hv.z, acc[b]);
        acc[b] = fmaf(w.w, hv.w, acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < GRU_ROWS; ++b) ghs[b * GRU_G + tid] = acc[b];
    __syncthreads();
    if (gate_thread) {
      const size_t row = (size_t)(b0 + gb) * T + t;
      const float *g = gi + row * GRU_G;
      const float *gh = ghs + gb * GRU_G;
      const float r = gru_sigmoid(g[gi_] + gh[gi_]);
      const float z = gru_sigmoid(g[GRU_H + gi_] + gh[GRU_H + gi_]);
      const float hn = gh[2 * GRU_H + gi_];
      const float n = tanhf(fmaf(r, hn, g[2 * GRU_H + gi_]));
      const float hp = hs[gb * GRU_H + gi_];
      const float h = fmaf(z, hp - n, n);                         // (1 - z) n + z h
      h_out[row * GRU_H + gi_] = h;
      if (save) {
        float *s = save + row * 5 * GRU_H + gi_;
        s[0] = r;
        s[GRU_H] = z;
        s[2 * GRU_H] = n;
        s[3 * GRU_H] = hn;
        s[4 * GRU_H] = hp;
      }
      hs[gb * GRU_H + gi_] = h;          // every thread finished reading h (sync above); only this thread reads it here
    }
    __syncthreads();
  }
}

// Reverse-time recurrence. dh_t = dy_t + z_{t+1} dh_{t+1} + W_hh^T dgh_{t+1};
//   dn = dh (1 - z), dz = dh (h_prev - n), dgn = dn (1 - n^2), dr = dgn hn
//   dgi = (dr r (1 - r), dz z (1 - z), dgn),  dgh = (same r, z parts, dgn r)
// smem: W[j][i] (thread i of a 128-wide chunk reads consecutive words), dgh[ROWS][3H], part[3][ROWS][H]
__global__ void __launch_bounds__(GRU_G, 1)
gru_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ save, const float *__restrict__ w_hh,
               float *__restrict__ dgi, float *__restrict__ dgh, int B, int T) {
  extern __shared__ float smem[];
  float *W = smem;                                 // [3H][H]
  float *dghs = W + GRU_G * GRU_H;                  // [ROWS][3H]
  float *part = dghs + GRU_ROWS * GRU_G;            // [3][ROWS][H]
  const int tid = threadIdx.x;
  const int b0 = blockIdx.x * GRU_ROWS;
  for (int idx = tid; idx < GRU_G * GRU_H / 4; idx += GRU_G)
    reinterpret_cast<float4 *>(W)[idx] = reinterpret_cast<const float4 *>(w_hh)[idx];
  const int gb = tid / GRU_H, gi_ = tid % GRU_H;
  const bool gate_thread = tid < GRU_ROWS * GRU_H;
  const bool valid = gate_thread && b0 + gb < B;
  const int chunk = tid / GRU_H;                    // matvec phase: j in [chunk*H, chunk*H + H)
  float carry = 0.f;                                // dh flowing into step t from step t + 1
  __syncthreads();
  for (int t = T - 1; t >= 0; --t) {
    float dh = 0.f, z = 0.f;
    if (gate_thread) {
      float d_r = 0.f, d_z = 0.f, d_n = 0.f, r = 0.f;
      if (valid) {
        const size_t row = (size_t)(b0 + gb) * T + t;
        const float *s = save + row * 5 * GRU_H + gi_;
        r = s[0];
        z = s[GRU_H];
        const float n = s[2 * GRU_H], hn = s[3 * GRU_H], hp = s[4 * GRU_H];
        dh = dy[row * GRU_H + gi_] + carry;
        const float dn = dh * (1.f - z);
        const float dz = dh * (hp - n);
        d_n = dn * (1.f - n * n);
        const float dr = d_n * hn;
        d_r = dr * r * (1.f - r);
        d_z = dz * z * (1.f - z);
        float *a = dgi + row * GRU_G + gi_;
        a[0] = d_r;
        a[GRU_H] = d_z;
        a[2 * GRU_H] = d_n;
        float *c = dgh + row * GRU_G + gi_;
        c[0] = d_r;
        c[GRU_H] = d_z;
        c[2 * GRU_H] = d_n * r;
      }
      float *q = dghs + gb * GRU_G + gi_;
      q[0] = d_r;
      q[GRU_H] = d_z;
      q[2 * GRU_H] = d_n * r;
    }
    __syncthreads();
    {
      const float *Wc = W + (size_t)chunk * GRU_H * GRU_H + gi_;
      float acc[GRU_ROWS];
#pragma unroll
      for (int b = 0; b < GRU_ROWS; ++b) acc[b] = 0.f;
#pragma unroll 4
      for (int j = 0; j < GRU_H; ++j) {
        const float w = Wc[j * GRU_H];
#pragma unroll
        for (int b = 0; b < GRU_ROWS; ++b) acc[b] = fmaf(w, dghs[b * GRU_G + chunk * GRU_H + j], acc[b]);
      }
#pragma unroll
      for (int b = 0; b < GRU_ROWS; ++b) part[(chunk * GRU_ROWS + b) * GRU_H + gi_] = acc[b];
    }
    __syncthreads();
    if (gate_thread) {
      const float *p = part + gb * GRU_H + gi_;
      carry = fmaf(dh, z, (p[0] + p[GRU_ROWS * GRU_H]) + p[2 * GRU_ROWS * GRU_H]);
    }
    // the next iteration writes dghs only after this barrier pair: every thread has read it (matvec) and part is
    // consumed by its own writer's row before the next matvec overwrites it (after the next first barrier)
  }
}

constexpr int GM_TILE = 64, GM_BK = 16;

// C[m][n] (+)= sum_k A[m*sam + k*sak] * Bm[k*sbk + n*sbn]; split z covers k in [z*kc, min(K, (z+1)*kc)).
// out: split-K partials [S][M][N] (S > 1) or C itself; rs: row sums of A over the split (bias gradients), or null.
__global__ void __launch_bounds__(256)
gemm_f32_kernel(const float *__restrict__ A, long sam, long sak, const float *__restrict__ Bm, long sbk, long sbn,
                const float *__restrict__ bias, float *__restrict__ out, long ldc, float *__restrict__ rs, int M, int N,
                int K, int kc) {
  __shared__ float As[GM_BK][GM_TILE + 4];
  __shared__ float Bs[GM_BK][GM_TILE + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * GM_TILE, n0 = blockIdx.x * GM_TILE;
  const int k_begin = blockIdx.z * kc, k_end = min(K, k_begin + kc);
  const bool do_rs = rs != nullptr && blockIdx.x == 0;
  float acc[4][4] = {};
  float rsum = 0.f;
  for (int k0 = k_begin; k0 < k_end; k0 += GM_BK) {
    for (int e = tid; e < GM_BK * GM_TILE; e += 256) {
      // A: consecutive threads walk m when A is m-contiguous, k otherwise
      int kk, mm;
      if (sam == 1) { mm = e % GM_TILE; kk = e / GM_TILE; } else { kk = e % GM_BK; mm = e / GM_BK; }
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < M && k < k_end) ? A[(long)m * sam + (long)k * sak] : 0.f;
      int kb, nn;
      if (sbn == 1) { nn = e % GM_TILE; kb = e / GM_TILE; } else { kb = e % GM_BK; nn = e / GM_BK; }
      const int n = n0 + nn, k2 = k0 + kb;
      Bs[kb][nn] = (n < N && k2 < k_end) ? Bm[(long)k2 * sbk + (long)n * sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GM_BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (do_rs && tid < GM_TILE) {
#pragma unroll
      for (int kk = 0; kk < GM_BK; ++kk) rsum += As[kk][tid];
    }
    __syncthreads();
  }
  const bool split = gridDim.z > 1;
  float *o = split ? out + (size_t)blockIdx.z * M * N : out;
  const long ld = split ? N : ldc;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + 16 * i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n < N) o[(long)m * ld + n] = acc[i][j] + ((!split && bias) ? bias[n] : 0.f);
    }
  }
  if (do_rs && tid < GM_TILE && m0 + tid < M) rs[(size_t)blockIdx.z * M + m0 + tid] = rsum;
}

// fixed-order sum of the S split-K partials (and of the row-sum partials)
__global__ void __launch_bounds__(256)
gemm_f32_reduce_kernel(const float *__restrict__ part, const float *__restrict__ bias, float *__restrict__ C, long ldc,
                       const float *__restrict__ rs_part, float *__restrict__ rs, int M, int N, int S) {
  const long total = (long)M * N;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < total + (rs ? M : 0); i += (long)gridDim.x * 256) {
    if (i < total) {
      float t = 0.f;
      for (int s = 0; s < S; ++s) t += part[(size_t)s * total + i];
      const int m = (int)(i / N), n = (int)(i % N);
      C[(long)m * ldc + n] = t + (bias ? bias[n] : 0.f);
    } else {
      const int m = (int)(i - total);
      float t = 0.f;
      for (int s = 0; s < S; ++s) t += rs_part[(size_t)s * M + m];
      rs[m] = t;
    }
  }
}

}  // namespace rave

extern "C" int rave_gru_fwd(const float *gi, const float *w_hh, const float *b_hh, float *h_out, float *save, int B,
                            int T, int H, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(gi && w_hh && b_hh && h_out && B > 0 && T > 0, "gru_fwd: bad argument");
  RAVE_CHECK_ARG(H == GRU_H, "gru_fwd: hidden size %d (the kernel is built for %d)", H, GRU_H);
  const size_t smem = (size_t)GRU_G * GRU_H * 4 + (size_t)GRU_ROWS * (GRU_H + GRU_G) * 4;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      set_error("gru_fwd: cannot reserve %zu bytes of shared memory", smem);
      return 2;
    }
    attr = true;
  }
  gru_fwd_kernel<<<ceil_div(B, GRU_ROWS), GRU_G, smem, (cudaStream_t)stream>>>(gi, w_hh, b_hh, h_out, save, B, T);
  RAVE_CHECK_LAUNCH("gru_fwd");
  return 0;
}

extern "C" int rave_gru_bwd(const float *dy, const float *save, const float *w_hh, float *dgi, float *dgh, int B, int T,
                            int H, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(dy && save && w_hh && dgi && dgh && B > 0 && T > 0, "gru_bwd: bad argument");
  RAVE_CHECK_ARG(H == GRU_H, "gru_bwd: hidden size %d (the kernel is built for %d)", H, GRU_H);
  const size_t smem = (size_t)GRU_G * GRU_H * 4 + (size_t)GRU_ROWS * GRU_G * 4 + (size_t)3 * GRU_ROWS * GRU_H * 4;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      set_error("gru_bwd: cannot reserve %zu bytes of shared memory", smem);
      return 2;
    }
    attr = true;
  }
  gru_bwd_kernel<<<ceil_div(B, GRU_ROWS), GRU_G, smem, (cudaStream_t)stream>>>(dy, save, w_hh, dgi, dgh, B, T);
  RAVE_CHECK_LAUNCH("gru_bwd");
  return 0;
}

extern "C" int rave_gemm_f32_splits(int M, int N, int K) {
  const int tiles = rave::ceil_div(M, rave::GM_TILE) * rave::ceil_div(N, rave::GM_TILE);
  int s = rave::ceil_div(264, tiles);                 // about two waves of CTAs on 132 SMs
  if (s > K / 256) s = K / 256;                      // each split keeps >= 256 k
  if (s > 16) s = 16;
  return s < 1 ? 1 : s;
}

extern "C" int rave_gemm_f32(const float *A, long sam, long sak, const float *Bm, long sbk, long sbn, const float *bias,
                             float *C, long ldc, float *rowsum, int M, int N, int K, float *ws, int splits,
                             void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(A && Bm && C && M > 0 && N > 0 && K > 0 && splits >= 1 && (splits == 1 || ws),
                 "gemm_f32: bad argument");
  int kc = ceil_div(ceil_div(K, splits), GM_BK) * GM_BK;
  const int S = ceil_div(K, kc);
  dim3 grid(ceil_div(N, GM_TILE), ceil_div(M, GM_TILE), S);
  if (S == 1) {
    gemm_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, sam, sak, Bm, sbk, sbn, bias, C, ldc, rowsum, M, N, K,
                                                             kc);
    RAVE_CHECK_LAUNCH("gemm_f32");
    return 0;
  }
  // workspace: [S][M][N] partials, then [S][M] row-sum partials
  float *rs_part = rowsum ? ws + (size_t)S * M * N : nullptr;
  gemm_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, sam, sak, Bm, sbk, sbn, nullptr, ws, N, rs_part, M, N, K,
                                                           kc);
  RAVE_CHECK_LAUNCH("gemm_f32");
  const long total = (long)M * N + (rowsum ? M : 0);
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  gemm_f32_reduce_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(ws, bias, C, ldc, rs_part, rowsum, M, N, S);
  RAVE_CHECK_LAUNCH("gemm_f32_reduce");
  return 0;
}
