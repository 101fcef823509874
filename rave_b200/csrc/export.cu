// The exported model's latent arithmetic (scripts/export.py:351-408, rave/blocks.py:933-963), per frame of a [B][C][T]
// latent:
//   latent_project   : VariationalScriptedRAVE.post_process_latent (reparametrise, centre, first l PCA rows)
//   latent_unproject : VariationalScriptedRAVE.pre_process_latent (latent_pca^T [z ; noise] + latent_mean)
//   rvq_encode       : ResidualVectorQuantization.encode, all Q stages in one launch (DiscreteScriptedRAVE)
//   rvq_decode       : clamp + truncate the float codes, sum the codebook rows, append the noise channels
//   sphere_to_angles / angles_to_sphere : unit_norm_vector_to_angles / angles_to_unit_norm_vector
// Everything is fp32 and every sum is added in a fixed order (no float atomics): two runs give the same bits.
#include "common.cuh"

namespace rave {

constexpr int EX_THREADS = 256;

inline int ex_blocks(long n) { return (int)((n + EX_THREADS - 1) / EX_THREADS); }

// out[b][i][t] = sum_c pca[i][c] centred_sample(z[b][c][t], z[b][L + c][t], eps[b][c][t], latent_mean[c]), i < l.
// One thread per output, t fastest (coalesced); the sample is recomputed by the l threads that read it.
__global__ void __launch_bounds__(EX_THREADS)
latent_project_kernel(const float *__restrict__ z, const float *__restrict__ eps, const float *__restrict__ lmean,
                      const float *__restrict__ pca, float *__restrict__ out, int B, int L, int T, int l) {
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= (long)B * l * T) return;
  const int t = (int)(n % T), i = (int)((n / T) % l), b = (int)(n / ((long)T * l));
  const float *zm = z + (size_t)b * 2 * L * T + t, *zs = zm + (size_t)L * T, *ep = eps + (size_t)b * L * T + t;
  const float *row = pca + (size_t)i * L;
  float acc = 0.f;
  for (int c = 0; c < L; ++c)
    acc = fmaf(row[c], centred_sample(zm[(size_t)c * T], zs[(size_t)c * T], ep[(size_t)c * T], lmean[c]), acc);
  out[n] = acc;
}

// out[b][c][t] = sum_j pca[j][c] y[j] + latent_mean[c], y = [z[b][:, t] ; noise[b][:, t]] (l + (L - l) rows).
__global__ void __launch_bounds__(EX_THREADS)
latent_unproject_kernel(const float *__restrict__ z, const float *__restrict__ noise, const float *__restrict__ lmean,
                        const float *__restrict__ pca, float *__restrict__ out, int B, int L, int T, int l) {
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= (long)B * L * T) return;
  const int t = (int)(n % T), c = (int)((n / T) % L), b = (int)(n / ((long)T * L));
  const float *zp = z + (size_t)b * l * T + t, *np = noise + (size_t)b * (L - l) * T + t;
  float acc = 0.f;
  for (int j = 0; j < l; ++j) acc = fmaf(pca[(size_t)j * L + c], zp[(size_t)j * T], acc);
  for (int j = l; j < L; ++j) acc = fmaf(pca[(size_t)j * L + c], np[(size_t)(j - l) * T], acc);
  out[n] = __fadd_rn(acc, lmean[c]);
}

// ---------------------------------------------------------------------------------------------------------------------
// Residual vector quantisation.  A CTA owns RVQ_F frames (rows n = b T + t) and keeps their residuals in shared memory
// for all Q stages.  Each stage streams the stage's codebook through shared memory in tiles of RVQ_KT codes, double
// buffered with cp.async, and scores every (frame, code) pair of the tile: thread (ty, tx) owns frames ty + 8 i and codes
// tx + 16 j (i, j < 4), a 4 x 4 block of dot products added over d in order.  The distance is the reference's expanded
// form |r|^2 - 2 r.c + |c|^2; |c|^2 comes from `norms` [Q][K], written by rvq_norms_kernel just before.  The 16
// threads of a frame reduce their (distance, code) minima with shuffles, ties to the lowest code; the residual then
// loses the chosen row (read from L2) and the next stage begins.
constexpr int RVQ_F = 32;
constexpr int RVQ_KT = 64;
constexpr int RVQ_THREADS = 128;
constexpr int RVQ_MAX_D = 256;

__global__ void __launch_bounds__(EX_THREADS)
rvq_norms_kernel(const float *__restrict__ cb, float *__restrict__ norms, long QK, int D) {
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= QK) return;
  const float *c = cb + (size_t)n * D;
  float acc = 0.f;
  for (int d = 0; d < D; ++d) acc = fmaf(c[d], c[d], acc);
  norms[n] = acc;
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

inline size_t rvq_smem_bytes(int D) {
  const int P = D + 4;
  return ((size_t)RVQ_F * P + 2 * (size_t)RVQ_KT * P + 2 * RVQ_KT + 2 * RVQ_F) * sizeof(float);
}

// codebook tile k0 .. k0 + RVQ_KT - 1 of stage q (rows past K are zero-filled) and its norms
__device__ __forceinline__ void rvq_load_tile(float *tile, float *tnorm, const float *__restrict__ cbq,
                                              const float *__restrict__ nq, int k0, int K, int D) {
  const int P = D + 4, D4 = D / 4;
  for (int idx = threadIdx.x; idx < RVQ_KT * D4; idx += RVQ_THREADS) {
    const int r = idx / D4, c4 = idx - r * D4, k = k0 + r;
    const bool ok = k < K;
    cp_async16(tile + r * P + 4 * c4, ok ? cbq + (size_t)k * D + 4 * c4 : cbq, ok ? 16 : 0);
  }
  if (threadIdx.x < RVQ_KT) {
    const int k = k0 + threadIdx.x;
    cp_async4(tnorm + threadIdx.x, k < K ? nq + k : nq, k < K ? 4 : 0);
  }
  cp_async_commit();
}

__global__ void __launch_bounds__(RVQ_THREADS)
rvq_encode_kernel(const float *__restrict__ x, const float *__restrict__ cb, const float *__restrict__ norms,
                  int *__restrict__ codes, int B, int D, int T, int Q, int K) {
  extern __shared__ __align__(16) float sm[];
  const int P = D + 4;
  float *res = sm;                                   // [RVQ_F][P]
  float *tiles = res + RVQ_F * P;                    // [2][RVQ_KT][P]
  float *tnorm = tiles + 2 * RVQ_KT * P;             // [2][RVQ_KT]
  float *rr = tnorm + 2 * RVQ_KT;                    // [RVQ_F]
  int *sel = reinterpret_cast<int *>(rr + RVQ_F);    // [RVQ_F]
  const long N = (long)B * T, n0 = (long)blockIdx.x * RVQ_F;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

  for (int idx = tid; idx < RVQ_F * D; idx += RVQ_THREADS) {
    const int f = idx % RVQ_F, d = idx / RVQ_F;
    const long n = n0 + f;
    float v = 0.f;
    if (n < N) {
      const long b = n / T, t = n - b * T;
      v = x[((size_t)b * D + d) * T + t];
    }
    res[f * P + d] = v;
  }
  const int n_tiles = (K + RVQ_KT - 1) / RVQ_KT;

  for (int q = 0; q < Q; ++q) {
    const float *cbq = cb + (size_t)q * K * D, *nq = norms + (size_t)q * K;
    rvq_load_tile(tiles, tnorm, cbq, nq, 0, K, D);
    __syncthreads();                                 // residuals of the previous stage are final
    if (tid < RVQ_F) {
      float a = 0.f;
      for (int d = 0; d < D; ++d) a = fmaf(res[tid * P + d], res[tid * P + d], a);
      rr[tid] = a;
    }
    float best[4];
    int bestk[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      best[i] = INFINITY;
      bestk[i] = 0x7fffffff;
    }
    for (int kt = 0; kt < n_tiles; ++kt) {
      const int buf = kt & 1;
      if (kt + 1 < n_tiles) {
        rvq_load_tile(tiles + (buf ^ 1) * RVQ_KT * P, tnorm + (buf ^ 1) * RVQ_KT, cbq, nq, (kt + 1) * RVQ_KT, K, D);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      const float *tl = tiles + buf * RVQ_KT * P;
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 2
      for (int d = 0; d < D; d += 4) {
        float4 r[4], c[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) r[i] = *reinterpret_cast<const float4 *>(res + (ty + 8 * i) * P + d);
#pragma unroll
        for (int j = 0; j < 4; ++j) c[j] = *reinterpret_cast<const float4 *>(tl + (tx + 16 * j) * P + d);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[i][j] = fmaf(r[i].x, c[j].x, acc[i][j]);
            acc[i][j] = fmaf(r[i].y, c[j].y, acc[i][j]);
            acc[i][j] = fmaf(r[i].z, c[j].z, acc[i][j]);
            acc[i][j] = fmaf(r[i].w, c[j].w, acc[i][j]);
          }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = kt * RVQ_KT + tx + 16 * j;
        if (k >= K) continue;
        const float cn = tnorm[buf * RVQ_KT + tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float dist = __fadd_rn(__fsub_rn(rr[ty + 8 * i], 2.f * acc[i][j]), cn);
          if (dist < best[i]) {      // a thread meets its codes in increasing order: ties keep the lowest
            best[i] = dist;
            bestk[i] = k;
          }
        }
      }
      __syncthreads();                               // the buffer is refilled by the next iteration's prefetch
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {              // the 16 threads of frame ty + 8 i are one half-warp
        const float od = __shfl_xor_sync(0xffffffffu, best[i], o);
        const int ok = __shfl_xor_sync(0xffffffffu, bestk[i], o);
        if (od < best[i] || (od == best[i] && ok < bestk[i])) {
          best[i] = od;
          bestk[i] = ok;
        }
      }
      if (tx == 0) sel[ty + 8 * i] = bestk[i] < K ? bestk[i] : 0;   // no finite distance (non-finite input): code 0
    }
    __syncthreads();
    if (tid < RVQ_F && n0 + tid < N) {
      const long n = n0 + tid, b = n / T, t = n - b * T;
      codes[((size_t)b * Q + q) * T + t] = sel[tid];
    }
    for (int idx = tid; idx < RVQ_F * D; idx += RVQ_THREADS) {
      const int f = idx / D, d = idx - f * D;
      res[f * P + d] = __fsub_rn(res[f * P + d], cbq[(size_t)sel[f] * D + d]);
    }
  }
}

// out[b][d][t] = sum_q cb[q][k_q][d] (added in q order from 0), k_q = trunc(clamp(codes[b][q][t], 0, K - 1)) (NaN
// gives code 0); out[b][D + j][t] = noise[b][j][t], j < Nn.
__global__ void __launch_bounds__(EX_THREADS)
rvq_decode_kernel(const float *__restrict__ codes, const float *__restrict__ cb, const float *__restrict__ noise,
                  float *__restrict__ out, int B, int Q, int T, int K, int D, int Nn) {
  const int C = D + Nn;
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= (long)B * C * T) return;
  const int t = (int)(n % T), c = (int)((n / T) % C), b = (int)(n / ((long)T * C));
  if (c >= D) {
    out[n] = noise[((size_t)b * Nn + (c - D)) * T + t];
    return;
  }
  const float top = (float)(K - 1);
  float acc = 0.f;
  for (int q = 0; q < Q; ++q) {
    float v = codes[((size_t)b * Q + q) * T + t];
    v = v < 0.f ? 0.f : v;                           // torch.clamp keeps NaN; the conversion below maps it to 0
    v = v > top ? top : v;
    const int k = (int)v;
    acc = __fadd_rn(acc, cb[((size_t)q * K + k) * D + c]);
  }
  out[n] = acc;
}

// ---------------------------------------------------------------------------------------------------------------------
// Hyperspherical angles, one thread per frame (b, t) of x [B][L][T] / angles [B][L-1][T].
constexpr float EX_PI = 3.14159265358979323846f;
constexpr float EX_TWO_PI = 6.28318530717958647692f;

// Tail norms s_i = sqrt(sum_{j >= i} x_j^2), the last two squares added first (as the reference's merge does), then
// x_{i} added to the running sum from the end.  angle_i = arccos(clamp(x_i / s_i, -1, 1)) (NaN kept), the last one
// reflected to 2 pi - angle when x_{L-1} < 0 (or NaN); angles / pi (the last / 2 pi), then 2 (a - 0.5).
__global__ void __launch_bounds__(EX_THREADS)
sphere_to_angles_kernel(const float *__restrict__ x, float *__restrict__ out, int B, int L, int T) {
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= (long)B * T) return;
  const long b = n / T, t = n - b * T;
  const float *xp = x + (size_t)b * L * T + t;
  float *op = out + (size_t)b * (L - 1) * T + t;
  const float last = xp[(size_t)(L - 1) * T];
  float s = __fmul_rn(last, last);
  for (int i = L - 2; i >= 0; --i) {
    const float xi = xp[(size_t)i * T];
    s = __fadd_rn(__fmul_rn(xi, xi), s);
    float c = __fdiv_rn(xi, sqrtf(s));
    c = c > 1.f ? 1.f : c;
    c = c < -1.f ? -1.f : c;
    float a = acosf(c);
    if (i == L - 2)
      a = __fdiv_rn(last >= 0.f ? a : __fsub_rn(EX_TWO_PI, a), EX_TWO_PI);
    else
      a = __fdiv_rn(a, EX_PI);
    op[(size_t)i * T] = __fmul_rn(2.f, __fsub_rn(a, 0.5f));
  }
}

// torch's floor remainder a % 1 (c10's remainder: fmod, then + 1 when the sign differs from the divisor's)
__device__ __forceinline__ float floor_mod1(float a) {
  float m = fmodf(a, 1.f);
  if (m != 0.f && m < 0.f) m = __fadd_rn(m, 1.f);
  return m;
}

// phi_i = ((a_i / 2 + 0.5) mod 1) pi (the last 2 pi); x_i = cos(phi_i) prod_{j < i} sin(phi_j), x_{L-1} = prod_j sin(phi_j)
__global__ void __launch_bounds__(EX_THREADS)
angles_to_sphere_kernel(const float *__restrict__ angles, float *__restrict__ out, int B, int L, int T) {
  const long n = blockIdx.x * (long)EX_THREADS + threadIdx.x;
  if (n >= (long)B * T) return;
  const long b = n / T, t = n - b * T;
  const float *ap = angles + (size_t)b * (L - 1) * T + t;
  float *op = out + (size_t)b * L * T + t;
  float prod = 1.f;
  for (int i = 0; i < L - 1; ++i) {
    const float u = floor_mod1(__fadd_rn(__fdiv_rn(ap[(size_t)i * T], 2.f), 0.5f));
    const float phi = __fmul_rn(u, i == L - 2 ? EX_TWO_PI : EX_PI);
    op[(size_t)i * T] = __fmul_rn(cosf(phi), prod);
    prod = __fmul_rn(prod, sinf(phi));
  }
  op[(size_t)(L - 1) * T] = prod;
}

}  // namespace rave

extern "C" int rave_latent_project(const float *z, const float *eps, const float *latent_mean, const float *latent_pca,
                                   float *out, int B, int L, int T, int l, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && eps && latent_mean && latent_pca && out, "latent_project: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && T > 0 && l > 0 && l <= L, "latent_project: bad shape (B %d, L %d, T %d, l %d)", B, L,
                 T, l);
  const long n = (long)B * l * T;
  latent_project_kernel<<<ex_blocks(n), EX_THREADS, 0, (cudaStream_t)stream>>>(z, eps, latent_mean, latent_pca, out, B,
                                                                               L, T, l);
  RAVE_CHECK_LAUNCH("latent_project");
  return 0;
}

extern "C" int rave_latent_unproject(const float *z, const float *noise, const float *latent_mean,
                                     const float *latent_pca, float *out, int B, int L, int T, int l, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && latent_mean && latent_pca && out && (noise || l == L), "latent_unproject: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && T > 0 && l > 0 && l <= L, "latent_unproject: bad shape (B %d, L %d, T %d, l %d)", B,
                 L, T, l);
  const long n = (long)B * L * T;
  latent_unproject_kernel<<<ex_blocks(n), EX_THREADS, 0, (cudaStream_t)stream>>>(z, noise, latent_mean, latent_pca, out,
                                                                                 B, L, T, l);
  RAVE_CHECK_LAUNCH("latent_unproject");
  return 0;
}

extern "C" int rave_rvq_encode(const float *x, const float *codebooks, float *norms, int *codes, int B, int D, int T,
                               int Q, int K, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && codebooks && norms && codes, "rvq_encode: null pointer");
  RAVE_CHECK_ARG(B > 0 && T > 0 && Q > 0 && K > 0 && D > 0 && D % 4 == 0 && D <= RVQ_MAX_D,
                 "rvq_encode: bad shape (B %d, D %d, T %d, Q %d, K %d); D must be a multiple of 4, at most %d", B, D, T,
                 Q, K, RVQ_MAX_D);
  RAVE_CHECK_ARG(((uintptr_t)codebooks & 15) == 0, "rvq_encode: codebooks must be 16-byte aligned");
  const cudaStream_t s = (cudaStream_t)stream;
  const long QK = (long)Q * K;
  rvq_norms_kernel<<<ex_blocks(QK), EX_THREADS, 0, s>>>(codebooks, norms, QK, D);
  RAVE_CHECK_LAUNCH("rvq_encode (norms)");
  const size_t smem = rvq_smem_bytes(D);
  if (cudaFuncSetAttribute(rvq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    cudaGetLastError();
    set_error("rvq_encode: %zu bytes of shared memory refused", smem);
    return 2;
  }
  const long frames = (long)B * T;
  rvq_encode_kernel<<<(int)((frames + RVQ_F - 1) / RVQ_F), RVQ_THREADS, smem, s>>>(x, codebooks, norms, codes, B, D, T,
                                                                                   Q, K);
  RAVE_CHECK_LAUNCH("rvq_encode");
  return 0;
}

extern "C" int rave_rvq_decode(const float *codes, const float *codebooks, const float *noise, float *out, int B, int Q,
                               int T, int K, int D, int n_noise, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(codes && codebooks && out && (noise || n_noise == 0), "rvq_decode: null pointer");
  RAVE_CHECK_ARG(B > 0 && Q > 0 && T > 0 && K > 0 && D > 0 && n_noise >= 0,
                 "rvq_decode: bad shape (B %d, Q %d, T %d, K %d, D %d, noise %d)", B, Q, T, K, D, n_noise);
  const long n = (long)B * (D + n_noise) * T;
  rvq_decode_kernel<<<ex_blocks(n), EX_THREADS, 0, (cudaStream_t)stream>>>(codes, codebooks, noise, out, B, Q, T, K, D,
                                                                           n_noise);
  RAVE_CHECK_LAUNCH("rvq_decode");
  return 0;
}

extern "C" int rave_sphere_to_angles(const float *x, float *angles, int B, int L, int T, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && angles, "sphere_to_angles: null pointer");
  RAVE_CHECK_ARG(B > 0 && L >= 2 && T > 0, "sphere_to_angles: bad shape (B %d, L %d, T %d)", B, L, T);
  sphere_to_angles_kernel<<<ex_blocks((long)B * T), EX_THREADS, 0, (cudaStream_t)stream>>>(x, angles, B, L, T);
  RAVE_CHECK_LAUNCH("sphere_to_angles");
  return 0;
}

extern "C" int rave_angles_to_sphere(const float *angles, float *x, int B, int L, int T, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(angles && x, "angles_to_sphere: null pointer");
  RAVE_CHECK_ARG(B > 0 && L >= 2 && T > 0, "angles_to_sphere: bad shape (B %d, L %d, T %d)", B, L, T);
  angles_to_sphere_kernel<<<ex_blocks((long)B * T), EX_THREADS, 0, (cudaStream_t)stream>>>(angles, x, B, L, T);
  RAVE_CHECK_LAUNCH("angles_to_sphere");
  return 0;
}
