// Latent regularisers of the v2 "Regularization" options (rave/blocks.py:748-791, 833-849):
//   WasserteinEncoder: the MMD between the encoder's latent rows and a standard normal prior sample, with the kernel
//     k(a, b) = exp(-|a - b|^2 / D^2)   (rave/blocks.py:761-763: `.pow(2).mean(2) / D`),
//   SphericalEncoder: z / |z| per (b, t) column.
// Everything is fp32 and every sum is added in a fixed order (no float atomics): two runs give the same bits.
#include "common.cuh"

namespace rave {

constexpr int MMD_DC = 8;            // latent dimensions per shared-memory chunk; D is padded to MMD_DC * NC with zeros
constexpr int MMD_FWD_T = 64;        // forward tile: 64 x 64 row pairs, 4 x 4 per thread
constexpr int MMD_BWD_T = 32;        // backward tile: 32 i-rows x 32 j-rows
constexpr int MMD_THREADS = 256;
constexpr int MMD_MAX_NC = 8;        // D <= 64
constexpr int MMD_MAX_ROWS = 65536;  // N = B * L: the forward's (N / 64)^2 CTAs and their partials stay bounded

// Row i = b * L + t of the latent z [B][D][L] (read in place: no permute copy) or of the prior sample y [N][D].
__device__ __forceinline__ float latent_row(const float *__restrict__ z, int i, int d, int D, int L) {
  const int b = i / L, t = i - b * L;
  return z[((size_t)b * D + d) * L + t];
}

// Fixed-order block sum of 256 threads: warp xor trees, then the 8 warp sums in warp order.  Returns the sum in every
// thread.  `red` holds 8 floats.
__device__ __forceinline__ float mmd_block_sum(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < MMD_THREADS / 32; ++w) s += red[w];
  return s;
}

// Grid (i-tiles, j-tiles): each CTA sums the three kernels over its 64 x 64 pairs, stores the three partials, and the
// last CTA to arrive adds every CTA's partials in block order and writes
//   means = (mean k(x, x), mean k(y, y), mean k(x, y)),   mmd = means[0] + means[1] - 2 means[2].
template <int NC>
__global__ void __launch_bounds__(MMD_THREADS)
mmd_fwd_kernel(const float *__restrict__ z, const float *__restrict__ y, float *__restrict__ means,
               float *__restrict__ mmd, int N, int D, int L, float inv_d2, float inv_nn, float *__restrict__ part,
               unsigned *__restrict__ ticket) {
  __shared__ __align__(16) float sxi[MMD_DC][MMD_FWD_T], sxj[MMD_DC][MMD_FWD_T];
  __shared__ __align__(16) float syi[MMD_DC][MMD_FWD_T], syj[MMD_DC][MMD_FWD_T];
  __shared__ float red[MMD_THREADS / 32];
  __shared__ unsigned is_last;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int i0 = blockIdx.x * MMD_FWD_T, j0 = blockIdx.y * MMD_FWD_T;
  float dxx[4][4] = {}, dyy[4][4] = {}, dxy[4][4] = {};
#pragma unroll 1
  for (int c = 0; c < NC; ++c) {
#pragma unroll
    for (int k = 0; k < MMD_DC * MMD_FWD_T / MMD_THREADS; ++k) {
      const int e = tid + k * MMD_THREADS, r = e % MMD_FWD_T, dd = e / MMD_FWD_T, d = c * MMD_DC + dd;
      const int i = i0 + r, j = j0 + r;
      const bool dv = d < D;
      sxi[dd][r] = (dv && i < N) ? latent_row(z, i, d, D, L) : 0.f;
      sxj[dd][r] = (dv && j < N) ? latent_row(z, j, d, D, L) : 0.f;
      syi[dd][r] = (dv && i < N) ? y[(size_t)i * D + d] : 0.f;
      syj[dd][r] = (dv && j < N) ? y[(size_t)j * D + d] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int dd = 0; dd < MMD_DC; ++dd) {
      const float4 xi = *reinterpret_cast<const float4 *>(&sxi[dd][ty * 4]);
      const float4 xj = *reinterpret_cast<const float4 *>(&sxj[dd][tx * 4]);
      const float4 yi = *reinterpret_cast<const float4 *>(&syi[dd][ty * 4]);
      const float4 yj = *reinterpret_cast<const float4 *>(&syj[dd][tx * 4]);
      const float xa[4] = {xi.x, xi.y, xi.z, xi.w}, xb[4] = {xj.x, xj.y, xj.z, xj.w};
      const float ya[4] = {yi.x, yi.y, yi.z, yi.w}, yb[4] = {yj.x, yj.y, yj.z, yj.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const float p = xa[a] - xb[b], q = ya[a] - yb[b], s = xa[a] - yb[b];
          dxx[a][b] = fmaf(p, p, dxx[a][b]);
          dyy[a][b] = fmaf(q, q, dyy[a][b]);
          dxy[a][b] = fmaf(s, s, dxy[a][b]);
        }
    }
    __syncthreads();
  }
  float sxx = 0.f, syy = 0.f, sxy = 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      if (i0 + ty * 4 + a < N && j0 + tx * 4 + b < N) {
        sxx += expf(-dxx[a][b] * inv_d2);
        syy += expf(-dyy[a][b] * inv_d2);
        sxy += expf(-dxy[a][b] * inv_d2);
      }
  sxx = mmd_block_sum(sxx, red);
  syy = mmd_block_sum(syy, red);
  sxy = mmd_block_sum(sxy, red);
  const unsigned nb = gridDim.x * gridDim.y, blk = blockIdx.x + gridDim.x * blockIdx.y;
  if (tid == 0) {
    part[blk * 3 + 0] = sxx;
    part[blk * 3 + 1] = syy;
    part[blk * 3 + 2] = sxy;
    __threadfence();
    is_last = atomicAdd(ticket, 1u) == nb - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float t[3] = {0.f, 0.f, 0.f};
  for (unsigned b = tid; b < nb; b += MMD_THREADS)
#pragma unroll
    for (int q = 0; q < 3; ++q) t[q] += __ldcg(part + b * 3 + q);
#pragma unroll
  for (int q = 0; q < 3; ++q) t[q] = mmd_block_sum(t[q], red) * inv_nn;
  if (tid == 0) {
    means[0] = t[0];
    means[1] = t[1];
    means[2] = t[2];
    mmd[0] = t[0] + t[1] - 2.f * t[2];
  }
}

// Grid (i-tiles of 32 rows, j-splits).  CTA (bi, s) accumulates, for its 32 rows i and every dimension d,
//   sum_j k(x_i, x_j) (x_i - x_j)[d] - k(x_i, y_j) (x_i - y_j)[d]
// over the j-rows of split s (32-row tiles), and stores it to part[s][i][d]; mmd_bwd_reduce_kernel adds the splits.
template <int NC>
__global__ void __launch_bounds__(MMD_THREADS)
mmd_bwd_kernel(const float *__restrict__ z, const float *__restrict__ y, float *__restrict__ part, int N, int D, int L,
               float inv_d2, int tiles_per_split, int Np) {
  constexpr int DP = NC * MMD_DC, T = MMD_BWD_T;
  __shared__ __align__(16) float sxi[DP][T], sxj[DP][T], syj[DP][T];
  __shared__ float kxx[T][T + 1], kxy[T][T + 1];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int i0 = blockIdx.x * T;
  for (int e = tid; e < DP * T; e += MMD_THREADS) {
    const int r = e % T, d = e / T, i = i0 + r;
    sxi[d][r] = (d < D && i < N) ? latent_row(z, i, d, D, L) : 0.f;
  }
  float acc[NC] = {};
  const int jt0 = blockIdx.y * tiles_per_split;
  const int jt1 = min(jt0 + tiles_per_split, (N + T - 1) / T);
#pragma unroll 1
  for (int jt = jt0; jt < jt1; ++jt) {
    const int j0 = jt * T;
    __syncthreads();                                   // previous tile's readers are done
    for (int e = tid; e < DP * T; e += MMD_THREADS) {
      const int r = e % T, d = e / T, j = j0 + r;
      const bool v = d < D && j < N;
      sxj[d][r] = v ? latent_row(z, j, d, D, L) : 0.f;
      syj[d][r] = v ? y[(size_t)j * D + d] : 0.f;
    }
    __syncthreads();
    // the 32 x 32 kernel values, 2 x 2 per thread
    float pxx[2][2] = {}, pxy[2][2] = {};
#pragma unroll
    for (int d = 0; d < DP; ++d) {
      const float2 xi = *reinterpret_cast<const float2 *>(&sxi[d][ty * 2]);
      const float2 xj = *reinterpret_cast<const float2 *>(&sxj[d][tx * 2]);
      const float2 yj = *reinterpret_cast<const float2 *>(&syj[d][tx * 2]);
      const float xa[2] = {xi.x, xi.y}, xb[2] = {xj.x, xj.y}, yb[2] = {yj.x, yj.y};
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const float p = xa[a] - xb[b], s = xa[a] - yb[b];
          pxx[a][b] = fmaf(p, p, pxx[a][b]);
          pxy[a][b] = fmaf(s, s, pxy[a][b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const bool v = j0 + tx * 2 + b < N;
        kxx[ty * 2 + a][tx * 2 + b] = v ? expf(-pxx[a][b] * inv_d2) : 0.f;
        kxy[ty * 2 + a][tx * 2 + b] = v ? expf(-pxy[a][b] * inv_d2) : 0.f;
      }
    __syncthreads();
    // output (i, d) = (o % 32, o / 32), o = tid + 256 q: one d per warp, the 32 lanes on 32 rows
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      const int o = tid + q * MMD_THREADS, i = o % T, d = o / T;
      const float xv = sxi[d][i];
      float s = acc[q];
#pragma unroll 8
      for (int j = 0; j < T; ++j) s += kxx[i][j] * (xv - sxj[d][j]) - kxy[i][j] * (xv - syj[d][j]);
      acc[q] = s;
    }
  }
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int o = tid + q * MMD_THREADS, i = o % T, d = o / T;
    part[((size_t)blockIdx.y * Np + i0 + i) * DP + d] = acc[q];
  }
}

// dz[b][d][t] = g * coef * sum over the splits s (in order) of part[s][i][d],  i = b * L + t,  coef = -4 / (D^2 N^2).
// g is read from device memory (the upstream gradient of the MMD: no host read, graph-capturable).
__global__ void __launch_bounds__(256)
mmd_bwd_reduce_kernel(const float *__restrict__ part, const float *__restrict__ g, float *__restrict__ dz, int N, int D,
                      int L, int DP, int Np, int splits, float coef) {
  const long total = (long)N * D;
  const float scale = g[0] * coef;
  for (long o = blockIdx.x * 256L + threadIdx.x; o < total; o += (long)gridDim.x * 256) {
    const int t = (int)(o % L);
    const long r = o / L;
    const int d = (int)(r % D), b = (int)(r / D), i = b * L + t;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[((size_t)k * Np + i) * DP + d];
    dz[o] = scale * s;
  }
}

// z [B][C][L] -> out = z / |z|_2 over C per (b, t), norm [B][L] saved for the backward.
__global__ void __launch_bounds__(256)
sphere_norm_fwd_kernel(const float *__restrict__ z, float *__restrict__ out, float *__restrict__ norm, int B, int C,
                       int L) {
  const long col = blockIdx.x * 256L + threadIdx.x;
  if (col >= (long)B * L) return;
  const int b = (int)(col / L), t = (int)(col % L);
  const float *zc = z + (size_t)b * C * L + t;
  float s = 0.f;
  for (int c = 0; c < C; ++c) s = fmaf(zc[(size_t)c * L], zc[(size_t)c * L], s);
  const float n = sqrtf(s);
  float *oc = out + (size_t)b * C * L + t;
  for (int c = 0; c < C; ++c) oc[(size_t)c * L] = zc[(size_t)c * L] / n;
  norm[col] = n;
}

// dz = (g - zh (zh . g)) / |z|   with zh = z / |z| the forward output.
__global__ void __launch_bounds__(256)
sphere_norm_bwd_kernel(const float *__restrict__ g, const float *__restrict__ zh, const float *__restrict__ norm,
                       float *__restrict__ dz, int B, int C, int L) {
  const long col = blockIdx.x * 256L + threadIdx.x;
  if (col >= (long)B * L) return;
  const int b = (int)(col / L), t = (int)(col % L);
  const size_t base = (size_t)b * C * L + t;
  float dot = 0.f;
  for (int c = 0; c < C; ++c) dot = fmaf(zh[base + (size_t)c * L], g[base + (size_t)c * L], dot);
  const float n = norm[col];
  for (int c = 0; c < C; ++c) dz[base + (size_t)c * L] = (g[base + (size_t)c * L] - zh[base + (size_t)c * L] * dot) / n;
}

template <template <int> class F, typename... A>
int mmd_dispatch(int nc, A... args) {
  switch (nc) {
    case 1: return F<1>::run(args...);
    case 2: return F<2>::run(args...);
    case 3: return F<3>::run(args...);
    case 4: return F<4>::run(args...);
    case 5: return F<5>::run(args...);
    case 6: return F<6>::run(args...);
    case 7: return F<7>::run(args...);
    case 8: return F<8>::run(args...);
  }
  set_error("mmd: latent size above %d", MMD_DC * MMD_MAX_NC);
  return 1;
}

template <int NC>
struct MmdFwd {
  static int run(dim3 grid, const float *z, const float *y, float *means, float *mmd, int N, int D, int L, float inv_d2,
                 float inv_nn, float *part, unsigned *ticket, cudaStream_t s) {
    mmd_fwd_kernel<NC><<<grid, MMD_THREADS, 0, s>>>(z, y, means, mmd, N, D, L, inv_d2, inv_nn, part, ticket);
    return 0;
  }
};

template <int NC>
struct MmdBwd {
  static int run(dim3 grid, const float *z, const float *y, float *part, int N, int D, int L, float inv_d2, int tps,
                 int Np, cudaStream_t s) {
    mmd_bwd_kernel<NC><<<grid, MMD_THREADS, 0, s>>>(z, y, part, N, D, L, inv_d2, tps, Np);
    return 0;
  }
};

}  // namespace rave

extern "C" int rave_mmd_fwd(const float *z, const float *prior, float *means, float *mmd, int B, int D, int L,
                            void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && prior && means && mmd, "mmd_fwd: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && (long)B * L <= MMD_MAX_ROWS, "mmd_fwd: B * L = %ld rows outside 1..%d", (long)B * L,
                 MMD_MAX_ROWS);
  RAVE_CHECK_ARG(D > 0 && D <= MMD_DC * MMD_MAX_NC, "mmd_fwd: latent size %d outside 1..%d", D, MMD_DC * MMD_MAX_NC);
  const int N = B * L, tiles = ceil_div(N, MMD_FWD_T);
  const cudaStream_t s = (cudaStream_t)stream;
  BlockSum bs;
  if (int rc = block_sum_begin(&bs, (long)tiles * tiles, 3, s)) return rc;
  const float inv_d2 = (float)(1.0 / ((double)D * D)), inv_nn = (float)(1.0 / ((double)N * N));
  mmd_dispatch<MmdFwd>(ceil_div(D, MMD_DC), dim3(tiles, tiles), z, prior, means, mmd, N, D, L, inv_d2, inv_nn, bs.part,
                       bs.ticket, s);
  block_sum_end(bs, s);
  RAVE_CHECK_LAUNCH("mmd_fwd");
  return 0;
}

extern "C" int rave_mmd_bwd(const float *z, const float *prior, const float *g, float *dz, int B, int D, int L,
                            void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && prior && g && dz, "mmd_bwd: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && (long)B * L <= MMD_MAX_ROWS, "mmd_bwd: B * L = %ld rows outside 1..%d", (long)B * L,
                 MMD_MAX_ROWS);
  RAVE_CHECK_ARG(D > 0 && D <= MMD_DC * MMD_MAX_NC, "mmd_bwd: latent size %d outside 1..%d", D, MMD_DC * MMD_MAX_NC);
  const int N = B * L, nc = ceil_div(D, MMD_DC), DP = nc * MMD_DC;
  const int itiles = ceil_div(N, MMD_BWD_T), jtiles = itiles, Np = itiles * MMD_BWD_T;
  // enough j-splits for two CTAs per SM; each split is a run of whole 32-row j-tiles
  int splits = ceil_div(2 * 132, itiles);
  if (splits > jtiles) splits = jtiles;
  const int tps = ceil_div(jtiles, splits);
  splits = ceil_div(jtiles, tps);
  const cudaStream_t s = (cudaStream_t)stream;
  void *part = nullptr;
  if (cudaMallocAsync(&part, (size_t)splits * Np * DP * sizeof(float), s) != cudaSuccess) {
    set_error("mmd_bwd: cudaMallocAsync of %d x %d x %d partials failed", splits, Np, DP);
    return 2;
  }
  const float inv_d2 = (float)(1.0 / ((double)D * D));
  const float coef = (float)(-4.0 / ((double)D * D * (double)N * N));
  mmd_dispatch<MmdBwd>(nc, dim3(itiles, splits), z, prior, (float *)part, N, D, L, inv_d2, tps, Np, s);
  RAVE_CHECK_LAUNCH("mmd_bwd");
  long blocks = ((long)N * D + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  mmd_bwd_reduce_kernel<<<(int)blocks, 256, 0, s>>>((const float *)part, g, dz, N, D, L, DP, Np, splits, coef);
  cudaFreeAsync(part, s);
  RAVE_CHECK_LAUNCH("mmd_bwd_reduce");
  return 0;
}

extern "C" int rave_sphere_norm_fwd(const float *z, float *out, float *norm, int B, int C, int L, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && out && norm && B > 0 && C > 0 && L > 0, "sphere_norm_fwd: bad argument");
  const long cols = (long)B * L;
  sphere_norm_fwd_kernel<<<(int)((cols + 255) / 256), 256, 0, (cudaStream_t)stream>>>(z, out, norm, B, C, L);
  RAVE_CHECK_LAUNCH("sphere_norm_fwd");
  return 0;
}

extern "C" int rave_sphere_norm_bwd(const float *g, const float *out, const float *norm, float *dz, int B, int C, int L,
                                    void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(g && out && norm && dz && B > 0 && C > 0 && L > 0, "sphere_norm_bwd: bad argument");
  const long cols = (long)B * L;
  sphere_norm_bwd_kernel<<<(int)((cols + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, out, norm, dz, B, C, L);
  RAVE_CHECK_LAUNCH("sphere_norm_bwd");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Streaming latent moments for the validation PCA (rave/model.py:464-488): count, mean and centred scatter matrix of the
// rows x_(b,t) = z[b][0:D][t] of z [B][C][L], accumulated in fp64 into state = [n | mean[D] | M2[D*D]].
//   Pass 1: grid (row blocks, 64 x 64 tiles of M2).  CTA (k, tile) walks block k's rows twice in 32-row tiles staged in
//           shared memory as fp64 (loads coalesced along t): first the per-channel sums of its channels (one thread per
//           channel, rows in order), then the centred products of its M2 tile (4 x 4 entries per thread, rows in order).
//           Every CTA that needs a channel's mean computes it with the same sequence of additions, so the copies agree
//           bit for bit.  Results (n_k, m_k, M2_k) go to work.
//   Pass 2: state <- state (+) block 0 (+) block 1 (+) ... with Chan's update, d = m_k - m, M2 += M2_k + d d^T n n_k / n';
//           each CTA owns 256 entries of M2 and replays the same running-mean sequence.
// Every sum is sequential in a fixed order: bit-identical across runs, no float atomics, no host read.
// ---------------------------------------------------------------------------------------------
namespace rave {

constexpr int LM_THREADS = 256;
constexpr int LM_TILE = 64;          // M2 tile edge (channels)
constexpr int LM_ROWS = 32;          // rows staged per shared-memory tile
constexpr int LM_MAX_D = 256;
constexpr int LM_MIN_BLOCK = 256;    // rows per block at least ...
constexpr int LM_MAX_BLOCKS = 132;   // ... and at most one block per SM

__host__ __device__ inline long lm_rows_per_block(long N) {
  long r = (N + LM_MAX_BLOCKS - 1) / LM_MAX_BLOCKS;
  if (r < LM_MIN_BLOCK) r = LM_MIN_BLOCK;
  return (r + LM_ROWS - 1) / LM_ROWS * LM_ROWS;
}

// Stage rows [g0, g0 + nr) of channels [c0, c0 + 64) into s[r][c] as fp64 minus `sub` (nullptr: raw); rows past nr and
// channels past D are zero.
__device__ __forceinline__ void lm_stage(double (*s)[LM_TILE + 1], const float *__restrict__ z, long g0, int nr, int c0,
                                         int C, int L, int D, const double *sub) {
#pragma unroll
  for (int k = 0; k < LM_ROWS * LM_TILE / LM_THREADS; ++k) {
    const int e = threadIdx.x + k * LM_THREADS, r = e % LM_ROWS, c = e / LM_ROWS, ch = c0 + c;
    double v = 0.0;
    if (r < nr && ch < D) {
      const long g = g0 + r, b = g / L, t = g - b * L;
      v = (double)z[((size_t)b * C + ch) * L + t];
      if (sub) v -= sub[c];
    }
    s[r][c] = v;
  }
}

__global__ void __launch_bounds__(LM_THREADS)
latent_moments_block_kernel(const float *__restrict__ z, int C, int L, int D, long N, long rpb, int tiles,
                            const double *__restrict__ state, double *__restrict__ work) {
  __shared__ double sa[LM_ROWS][LM_TILE + 1], sb[LM_ROWS][LM_TILE + 1];
  __shared__ double ma[LM_TILE], mb[LM_TILE];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int ti = blockIdx.y / tiles, tj = blockIdx.y % tiles, ca = ti * LM_TILE, cb = tj * LM_TILE;
  const long r0 = blockIdx.x * rpb, r1 = min(N, r0 + rpb), nb = r1 - r0;
  const size_t rec = 1 + (size_t)D + (size_t)D * D;
  double *out = work + 1 + D + blockIdx.x * rec;
  if (blockIdx.x == 0 && blockIdx.y == 0)                       // pass 2 reads the incoming (n, mean) from here
    for (int i = tid; i < 1 + D; i += LM_THREADS) work[i] = state[i];
  // block means of the channels of this tile's rows (ca..) and columns (cb..)
  double s = 0.0;
  for (long g0 = r0; g0 < r1; g0 += LM_ROWS) {
    const int nr = (int)min((long)LM_ROWS, r1 - g0);
    lm_stage(sa, z, g0, nr, ca, C, L, D, nullptr);
    lm_stage(sb, z, g0, nr, cb, C, L, D, nullptr);
    __syncthreads();
    if (tid < 2 * LM_TILE)
      for (int r = 0; r < nr; ++r) s += tid < LM_TILE ? sa[r][tid] : sb[r][tid - LM_TILE];
    __syncthreads();
  }
  if (tid < LM_TILE) ma[tid] = s / (double)nb;
  else if (tid < 2 * LM_TILE) mb[tid - LM_TILE] = s / (double)nb;
  __syncthreads();
  if (tj == 0 && tid < LM_TILE && ca + tid < D) out[1 + ca + tid] = ma[tid];
  if (blockIdx.y == 0 && tid == 0) out[0] = (double)nb;
  // centred scatter of the tile
  double acc[4][4] = {};
  for (long g0 = r0; g0 < r1; g0 += LM_ROWS) {
    const int nr = (int)min((long)LM_ROWS, r1 - g0);
    lm_stage(sa, z, g0, nr, ca, C, L, D, ma);
    lm_stage(sb, z, g0, nr, cb, C, L, D, mb);
    __syncthreads();
    for (int r = 0; r < nr; ++r) {
      double a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        a[q] = sa[r][ty * 4 + q];
        b[q] = sb[r][tx * 4 + q];
      }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = fma(a[p], b[q], acc[p][q]);
    }
    __syncthreads();
  }
  double *M2 = out + 1 + D;
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = ca + ty * 4 + p, j = cb + tx * 4 + q;
      if (i < D && j < D) M2[(size_t)i * D + j] = acc[p][q];
    }
}

__global__ void __launch_bounds__(LM_THREADS)
latent_moments_merge_kernel(int D, int nblk, const double *__restrict__ work, double *__restrict__ state) {
  __shared__ double mean[LM_MAX_D], dl[LM_MAX_D];
  const int tid = threadIdx.x;
  const long e = (long)blockIdx.x * LM_THREADS + tid, DD = (long)D * D;
  const int i = (int)(e / D), j = (int)(e % D);
  const size_t rec = 1 + (size_t)D + (size_t)D * D;
  double n = work[0];
  if (tid < D) mean[tid] = work[1 + tid];
  double m2 = e < DD ? state[1 + D + e] : 0.0;
  for (int k = 0; k < nblk; ++k) {
    const double *blk = work + 1 + D + k * rec;
    const double nk = blk[0], nn = n + nk, f = nk / nn, w = n * nk / nn;
    __syncthreads();                                            // mean[] of the previous merge is final
    if (tid < D) dl[tid] = blk[1 + tid] - mean[tid];
    __syncthreads();
    if (e < DD) m2 += blk[1 + D + e] + dl[i] * dl[j] * w;
    if (tid < D) mean[tid] = fma(dl[tid], f, mean[tid]);
    n = nn;
  }
  if (e < DD) state[1 + D + e] = m2;
  __syncthreads();
  if (blockIdx.x == 0) {
    if (tid == 0) state[0] = n;
    if (tid < D) state[1 + tid] = mean[tid];
  }
}

}  // namespace rave

extern "C" long rave_latent_moments_workspace_bytes(int B, int L, int D) {
  using namespace rave;
  if (B <= 0 || L <= 0 || D <= 0 || D > LM_MAX_D) return 0;
  const long N = (long)B * L, nblk = (N + lm_rows_per_block(N) - 1) / lm_rows_per_block(N);
  return (long)sizeof(double) * (1 + D + nblk * (1 + D + (long)D * D));
}

extern "C" int rave_latent_moments(const float *z, int B, int C, int L, int D, double *state, double *work,
                                   void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(z && state && work, "latent_moments: null pointer");
  RAVE_CHECK_ARG(B > 0 && L > 0 && C > 0, "latent_moments: bad shape [%d][%d][%d]", B, C, L);
  RAVE_CHECK_ARG(D >= 1 && D <= LM_MAX_D && D <= C, "latent_moments: latent size %d outside 1..min(%d, C = %d)", D,
                 LM_MAX_D, C);
  const long N = (long)B * L, rpb = lm_rows_per_block(N);
  const int nblk = (int)((N + rpb - 1) / rpb), tiles = ceil_div(D, LM_TILE);
  const cudaStream_t s = (cudaStream_t)stream;
  latent_moments_block_kernel<<<dim3(nblk, tiles * tiles), LM_THREADS, 0, s>>>(z, C, L, D, N, rpb, tiles, state, work);
  RAVE_CHECK_LAUNCH("latent_moments_block");
  latent_moments_merge_kernel<<<ceil_div(D * D, LM_THREADS), LM_THREADS, 0, s>>>(D, nblk, work, state);
  RAVE_CHECK_LAUNCH("latent_moments_merge");
  return 0;
}
