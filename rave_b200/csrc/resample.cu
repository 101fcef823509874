// The export's resampler (rave/resampler.py): one phase-bank FIR over every row of a [rows][L_in] signal,
//   y[r][i P + p] = sum_{k < K} W[p][k] x[r][i S + k - pad],   x = 0 outside [0, L_in),
// P = 1, S = ratio for the anti-aliased decimation (to_model_sampling_rate) and P = ratio, S = 1 for the polyphase
// interpolation (from_model_sampling_rate), which writes the interleaved output directly.
//
// A CTA owns n_i = RS_THREADS / P * RS_R consecutive positions i of one row.  It stages the bank and the input window
// those positions read ((n_i - 1) S + K samples) in shared memory with coalesced loads, the window split into its S phases
// (xs[m % S][m / S]) so that the S-strided reads of neighbouring positions hit neighbouring banks.  Thread t owns
// phase p = t % P and positions q + j Q (q = t / P, Q = threads / P, j < RS_R): one tap weight feeds RS_R outputs, and for
// each j the CTA's outputs are contiguous in y, so every store is coalesced and every output is written once.  Each output
// is a chain of float32 FMAs over k in increasing order (DESIGN §5.12 measures it against float64 accumulation): no
// atomics, so the bits depend on neither the run nor the rows launched with it.
#include "common.cuh"

namespace rave {

constexpr int RS_THREADS = 256;
constexpr int RS_R = 8;                       // outputs per thread and phase
constexpr int RS_MAX_K = 64;
constexpr int RS_MAX_RATIO = 8;

__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const float *__restrict__ x, const float *__restrict__ w, float *__restrict__ y, int L_in, int n_pos,
                int P, int S, int K, int pad, int tiles_per_row) {
  extern __shared__ float smem[];
  const int Q = RS_THREADS / P;               // positions per j step
  const int n_i = Q * RS_R;                   // positions of this CTA
  const int U = n_i - 1 + (K + S - 1) / S;    // window samples per phase
  float *ws = smem;                           // [P][K]
  float *xs = smem + P * K;                   // [S][U]

  const long row = blockIdx.x / tiles_per_row;
  const int i0 = (int)(blockIdx.x - row * tiles_per_row) * n_i;
  const float *xr = x + (size_t)row * L_in;
  const long base = (long)i0 * S - pad;       // input index of window sample 0

  for (int n = threadIdx.x; n < P * K; n += RS_THREADS) ws[n] = w[n];
  const int win = U * S;
  for (int m = threadIdx.x; m < win; m += RS_THREADS) {
    const long g = base + m;
    xs[(m % S) * U + m / S] = (g >= 0 && g < L_in) ? xr[g] : 0.f;
  }
  __syncthreads();

  const int p = threadIdx.x % P, q = threadIdx.x / P;
  if (q >= Q) return;                         // RS_THREADS % P idle threads
  float acc[RS_R];
#pragma unroll
  for (int j = 0; j < RS_R; ++j) acc[j] = 0.f;
  const float *wp = ws + p * K;
  for (int k = 0, kp = 0, ku = 0; k < K; ++k) {
    const float wk = wp[k];
    const float *xk = xs + kp * U + q + ku;   // window sample (q + j Q) S + k
#pragma unroll
    for (int j = 0; j < RS_R; ++j) acc[j] = fmaf(wk, xk[j * Q], acc[j]);
    if (++kp == S) kp = 0, ++ku;
  }
  float *yr = y + (size_t)row * n_pos * P;
#pragma unroll
  for (int j = 0; j < RS_R; ++j) {
    const int i = i0 + q + j * Q;
    if (i < n_pos) yr[(size_t)i * P + p] = acc[j];
  }
}

}  // namespace rave

extern "C" int rave_resample(const float *x, const float *w, float *y, long long rows, int L_in, int n_pos, int P,
                             int S, int K, int pad, void *stream) {
  using namespace rave;
  RAVE_CHECK_ARG(x && w && y, "resample: null pointer");
  RAVE_CHECK_ARG(rows > 0 && L_in > 0 && n_pos > 0 && pad >= 0, "resample: bad shape (rows %lld, L_in %d, n_pos %d, "
                 "pad %d)", rows, L_in, n_pos, pad);
  RAVE_CHECK_ARG(P >= 1 && P <= RS_MAX_RATIO && S >= 1 && S <= RS_MAX_RATIO && K >= 1 && K <= RS_MAX_K,
                 "resample: P %d, S %d, K %d outside 1..%d, 1..%d, 1..%d", P, S, K, RS_MAX_RATIO, RS_MAX_RATIO,
                 RS_MAX_K);
  RAVE_CHECK_ARG((long long)n_pos * P <= 0x7fffffffLL, "resample: %d x %d outputs per row", n_pos, P);
  const int n_i = RS_THREADS / P * RS_R;
  const int tiles = ceil_div(n_pos, n_i);
  const long long blocks = rows * tiles;
  RAVE_CHECK_ARG(blocks <= 0x7fffffffLL, "resample: %lld CTAs", blocks);
  const int U = n_i - 1 + ceil_div(K, S);
  const size_t smem = (size_t)(P * K + S * U) * sizeof(float);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    attr = true;
  }
  resample_kernel<<<(unsigned)blocks, RS_THREADS, smem, (cudaStream_t)stream>>>(x, w, y, L_in, n_pos, P, S, K, pad,
                                                                                 tiles);
  RAVE_CHECK_LAUNCH("resample");
  return 0;
}
