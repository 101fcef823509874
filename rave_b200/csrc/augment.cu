// Training-batch transforms of the reference's get_dataset (rave/dataset.py:207-262) on the device, per example and in
// the reference's order: int16 decode, random crop, phase-mangling allpass (RandomApply p = .8 of
// random_phase_mangle(x, 20, 2000, .99, sr)), Dequantize(16), normalize_signal, the derivator and RandomMute.
//
// The allpass y[n] = b0 x[n] + b1 x[n-1] + b2 x[n-2] - a1 y[n-1] - a2 y[n-2] is a linear recurrence over the whole
// crop of each (b, c) row, with only B * C rows.  It runs as a chunked parallel scan in float64 over the state
// s[n] = (y[n], y[n-1]) = A s[n-1] + (w[n], 0), A = [[-a1, -a2], [1, 0]], w = the FIR half:
//   * a CTA owns 2048 samples of one row (8 consecutive samples per thread) and reads the FIR inputs x[n-1], x[n-2]
//     across its left edge from the input itself (zero before the crop start: lfilter's zero initial state);
//   * each thread runs its 8 samples from the zero state; a Kogge-Stone scan over the 256 threads with the powers
//     A^(8 d) gives every thread the zero-state response entering it and the chunk's end state (its aggregate);
//   * the CTA publishes its aggregate, then folds the aggregates of all its row's earlier chunks, always in chunk
//     order (Horner with A^2048), into the state entering the chunk.  The fold never uses another CTA's folded result,
//     so the arithmetic -- and every output bit -- is the same whichever CTA finishes first.  CTAs take their chunk
//     from an arrival ticket, so every chunk a CTA waits for belongs to a CTA that is already running;
//   * each thread reruns its 8 samples from its true incoming state and writes each output once.
// With normalize_signal the example's peak is needed before any output: pass 1 (the scan above, plus a max over the
// example) leaves the aggregates and the peak in the workspace, pass 2 folds the stored aggregates (no waiting),
// recomputes the chunk, scales and writes.  The max is an integer atomicMax on the bits of |x| >= 0: order-free.
//
// Dtype flow (numpy 2.3, as the reference runs): when the allpass ran, everything after it is float64 up to the final
// cast; when it was skipped, the dequantised sum is rounded to float32 (`x +=` on a float32 array) and
// normalize_signal's gain is computed and applied in float32.
#include "common.cuh"

namespace rave {

constexpr int kAugThreads = 256;
constexpr int kAugPer = 8;                          // consecutive samples per thread
constexpr int kAugChunk = kAugThreads * kAugPer;    // samples per CTA
constexpr int kAugLog2Threads = 8;
constexpr double kPoleAmp = 0.99;                   // random_phase_mangle(x, 20, 2000, .99, sr): pole magnitude

__host__ __device__ constexpr int aug_skew(int i) { return i + (i >> 5); }  // conflict-free 8-sample rows per thread

struct Mat2 {
  double a, b, c, d;  // [[a, b], [c, d]]
};
__device__ __forceinline__ Mat2 mat_mul(const Mat2 &x, const Mat2 &y) {
  return {x.a * y.a + x.b * y.c, x.a * y.b + x.b * y.d, x.c * y.a + x.d * y.c, x.c * y.b + x.d * y.d};
}

// Philox4x32-10 (Salmon et al., SC'11)
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const unsigned lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
// U[0, 1) with 53 random bits from two words
__device__ __forceinline__ double u53(unsigned hi, unsigned lo) {
  return ((double)(hi >> 5) * 67108864.0 + (double)(lo >> 6)) * 0x1p-53;
}

struct AugArgs {
  const void *raw;
  int raw_int16, B, C, L, N, K;       // raw [B][C][L]; out [B][C][N]; K chunks per row
  const double *draws;                // [B][4]: crop offset, allpass applied, omega, keep
  const long long *key;               // [2]: Philox seed, counter offset
  const double *noise;                // [B][C][N] uniforms replacing the Philox draw, or NULL
  float *out;
  int derivative;
  double *agg;                        // [B * C][K][2] chunk aggregates
  unsigned *flag;                     // [B * C][K] aggregate published
  unsigned *ticket;
  unsigned long long *peak;           // [B] bits of the example's max |x|
};

// Dequantize(16): x + U[0, 1) / 2^16, the uniform of element (b, c, n)
__device__ __forceinline__ double dq_noise(const AugArgs &p, int b, int c, long n, uint2 key, unsigned koff) {
  if (p.noise) return p.noise[((size_t)b * p.C + c) * p.N + n] * 0x1p-16;
  const uint4 r = philox4x32(make_uint4((unsigned)(n >> 1), (unsigned)c, (unsigned)b, koff), key);
  return (n & 1 ? u53(r.z, r.w) : u53(r.x, r.y)) * 0x1p-16;
}

__device__ __forceinline__ unsigned ld_acquire(const unsigned *f) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(unsigned *f, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(f), "r"(v) : "memory");
}

// MODE 0: one pass, writes the output (no normalisation).  MODE 1: the scan and the example's peak, no output.
// MODE 2: the scale pass after MODE 1 (stored aggregates, no ticket).
template <int MODE>
__global__ void __launch_bounds__(kAugThreads) augment_kernel(const AugArgs p) {
  __shared__ float xs[aug_skew(kAugChunk + 2) + 1];   // x at n0 - 2 + i, i < kAugChunk + 2 (then the output tile)
  __shared__ double sv[kAugThreads][2];
  __shared__ Mat2 pw[kAugLog2Threads + 1];            // A^(8 * 2^k); pw[8] = A^2048
  __shared__ double carry[2];
  __shared__ unsigned vid_s;

  const int t = threadIdx.x;
  unsigned vid = blockIdx.x;
  if (MODE != 2) {
    if (t == 0) vid_s = atomicAdd(p.ticket, 1u);
    __syncthreads();
    vid = vid_s;
  }
  const int row = (int)(vid / (unsigned)p.K), chunk = (int)(vid % (unsigned)p.K);
  const int b = row / p.C, c = row % p.C;
  const double *dr = p.draws + 4 * (size_t)b;
  const long span = (long)p.L - p.N;
  const long off = min(max((long)dr[0], 0L), span);
  const bool apply = dr[1] != 0.0;
  const double keep = dr[3];
  const long n0 = (long)chunk * kAugChunk;

  // decode: float32(int16) / 32767 as a float32 division (rave/dataset.py:76-77)
  const size_t rbase = (size_t)row * p.L + off;
  for (int i = t; i < kAugChunk + 2; i += kAugThreads) {
    const long n = n0 - 2 + i;
    float v = 0.f;
    if (n >= 0 && n < p.N)
      v = p.raw_int16 ? __fdiv_rn((float)static_cast<const short *>(p.raw)[rbase + n], 32767.f)
                      : static_cast<const float *>(p.raw)[rbase + n];
    xs[aug_skew(i)] = v;
  }
  __syncthreads();
  const int i0 = t * kAugPer;
  float x[kAugPer + 2];                // x[k] = input at n0 + i0 - 2 + k
#pragma unroll
  for (int k = 0; k < kAugPer + 2; ++k) x[k] = xs[aug_skew(i0 + k)];

  double v[kAugPer];                   // allpass output (applied) or the float32 input
  double vprev;                        // the same at n0 + i0 - 1
  if (apply) {
    // pole_to_z_filter(omega, .99) (rave/dataset.py:281-285): z0 = .99 e^{i omega}
    const double omega = dr[2];
    const double re = kPoleAmp * cos(omega), im = kPoleAmp * sin(omega);
    const double r = hypot(re, im);
    const double a2 = r * r, a1 = -2.0 * re;
    const double b0 = a2, b1 = a1;     // b2 = 1
    if (t == 0) {
      Mat2 m = {-a1, -a2, 1.0, 0.0};
#pragma unroll
      for (int k = 0; k < 3; ++k) m = mat_mul(m, m);   // A^8
      for (int k = 0; k <= kAugLog2Threads; ++k) {
        pw[k] = m;
        m = mat_mul(m, m);
      }
    }
    double w[kAugPer];
#pragma unroll
    for (int k = 0; k < kAugPer; ++k) w[k] = b0 * x[k + 2] + b1 * x[k + 1] + (double)x[k];
    double y1 = 0.0, y2 = 0.0;         // zero-state run over this thread's samples
#pragma unroll
    for (int k = 0; k < kAugPer; ++k) {
      const double y = w[k] - a1 * y1 - a2 * y2;
      y2 = y1;
      y1 = y;
    }
    __syncthreads();
    // inclusive scan e_t = sum_{i <= t} (A^8)^(t - i) v_i
    double e0 = y1, e1 = y2;
#pragma unroll
    for (int k = 0; k < kAugLog2Threads; ++k) {
      const int d = 1 << k;
      sv[t][0] = e0;
      sv[t][1] = e1;
      __syncthreads();
      if (t >= d) {
        const Mat2 m = pw[k];
        const double q0 = sv[t - d][0], q1 = sv[t - d][1];
        e0 += m.a * q0 + m.b * q1;
        e1 += m.c * q0 + m.d * q1;
      }
      __syncthreads();
    }
    sv[t][0] = e0;
    sv[t][1] = e1;
    __syncthreads();
    if (t == 0) {
      double *agg = p.agg + ((size_t)row * p.K) * 2;
      if (MODE != 2 && chunk + 1 < p.K) {
        agg[2 * chunk] = sv[kAugThreads - 1][0];
        agg[2 * chunk + 1] = sv[kAugThreads - 1][1];
        st_release(p.flag + (size_t)row * p.K + chunk, 1u);
      }
      // state entering the chunk: the aggregates of chunks 0 .. chunk-1 folded in chunk order
      const Mat2 q = pw[kAugLog2Threads];
      double s0 = 0.0, s1 = 0.0;
      for (int j = 0; j < chunk; ++j) {
        if (MODE != 2)
          while (ld_acquire(p.flag + (size_t)row * p.K + j) == 0u) __nanosleep(64);
        const double g0 = __ldcg(agg + 2 * j), g1 = __ldcg(agg + 2 * j + 1);
        const double n0s = q.a * s0 + q.b * s1 + g0, n1s = q.c * s0 + q.d * s1 + g1;
        s0 = n0s;
        s1 = n1s;
      }
      carry[0] = s0;
      carry[1] = s1;
    }
    __syncthreads();
    // state entering this thread: exclusive scan + (A^8)^t carry
    double s0 = t > 0 ? sv[t - 1][0] : 0.0, s1 = t > 0 ? sv[t - 1][1] : 0.0;
    Mat2 mt = {1.0, 0.0, 0.0, 1.0};
#pragma unroll
    for (int k = 0; k < kAugLog2Threads; ++k)
      if ((t >> k) & 1) mt = mat_mul(mt, pw[k]);
    const double c0 = carry[0], c1 = carry[1];
    s0 += mt.a * c0 + mt.b * c1;
    s1 += mt.c * c0 + mt.d * c1;
    vprev = s0;
#pragma unroll
    for (int k = 0; k < kAugPer; ++k) {
      const double y = w[k] - a1 * s0 - a2 * s1;
      s1 = s0;
      s0 = y;
      v[k] = y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < kAugPer; ++k) v[k] = (double)x[k + 2];
    vprev = (double)x[1];
  }

  // Dequantize(16), in place: the sum is rounded to float32 when x is the float32 input
  const uint2 key = make_uint2((unsigned)(unsigned long long)p.key[0], (unsigned)((unsigned long long)p.key[0] >> 32));
  const unsigned koff = (unsigned)p.key[1];
  const long nb = n0 + i0;
  double d[kAugPer];
#pragma unroll
  for (int k = 0; k < kAugPer; ++k) {
    const long n = nb + k;
    const double q = n < p.N ? dq_noise(p, b, c, n, key, koff) : 0.0;
    d[k] = apply ? __dadd_rn(v[k], q) : (double)__double2float_rn(__dadd_rn(v[k], q));
  }
  double dprev = 0.0;                  // the dequantised sample before this thread's first (0 before the crop start)
  if (p.derivative && nb > 0 && nb <= p.N) {
    const double q = dq_noise(p, b, c, nb - 1, key, koff);
    dprev = apply ? __dadd_rn(vprev, q) : (double)__double2float_rn(__dadd_rn(vprev, q));
  }

  if (MODE == 1) {
    double m = 0.0;
#pragma unroll
    for (int k = 0; k < kAugPer; ++k)
      if (nb + k < p.N) m = fmax(m, fabs(d[k]));
    unsigned long long bits = (unsigned long long)__double_as_longlong(m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bits = max(bits, __shfl_xor_sync(0xffffffffu, bits, o));
    if ((t & 31) == 0 && bits) atomicMax(p.peak + b, bits);
    return;
  }

  if (MODE == 2) {
    // normalize_signal (rave/dataset.py:196-204); a zero peak leaves x unchanged
    const double pk = __longlong_as_double((long long)p.peak[b]);
    if (pk != 0.0) {
      if (apply) {
        const double lp = 20.0 * log10(pk);
        const double g = -lp < 30.0 ? pow(10.0, __ddiv_rn(-lp, 20.0)) : 31.622776601683793;  // 10 ** (30 / 20)
#pragma unroll
        for (int k = 0; k < kAugPer; ++k) d[k] = __dmul_rn(d[k], g);
        dprev = __dmul_rn(dprev, g);
      } else {
        // float32 flow; log10 and the power correctly rounded (see DESIGN)
        const float lp = __fmul_rn(20.f, __double2float_rn(log10(pk)));
        const float g = -lp < 30.f ? __double2float_rn(pow(10.0, (double)__fdiv_rn(-lp, 20.f))) : 31.622776f;
#pragma unroll
        for (int k = 0; k < kAugPer; ++k) d[k] = (double)__fmul_rn((float)d[k], g);
        dprev = (double)__fmul_rn((float)dprev, g);
      }
    }
  }

  // derivator lfilter([.5, -.5], [1]) in float64, RandomMute, the final float32 cast
  float o[kAugPer];
#pragma unroll
  for (int k = 0; k < kAugPer; ++k) {
    double y = d[k];
    if (p.derivative) {
      y = __dadd_rn(0.5 * d[k], -0.5 * dprev);
      dprev = d[k];
    }
    o[k] = __double2float_rn(__dmul_rn(y, keep));
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kAugPer; ++k) xs[aug_skew(i0 + k)] = o[k];
  __syncthreads();
  float *dst = p.out + (size_t)row * p.N + n0;
  const int valid = (int)min((long)kAugChunk, (long)p.N - n0);
  for (int i = t; i < valid; i += kAugThreads) dst[i] = xs[aug_skew(i)];
}

}  // namespace rave

using namespace rave;

extern "C" int rave_augment(const void *raw, int raw_int16, int B, int C, int L, int N, const double *draws,
                            const long long *key, const double *noise, float *out, int normalize, int derivative,
                            void *stream) {
  RAVE_CHECK_ARG(raw && draws && key && out, "rave_augment: null pointer");
  RAVE_CHECK_ARG(B >= 1 && C >= 1 && N >= 1 && L >= N, "rave_augment: bad shape B=%d C=%d L=%d N=%d", B, C, L, N);
  const long rows = (long)B * C, K = (N + kAugChunk - 1) / kAugChunk;
  RAVE_CHECK_ARG(rows * K < (1L << 31), "rave_augment: %ld chunks exceed the grid", rows * K);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t peak_b = (size_t)B * 8, agg_b = (size_t)rows * K * 16, flag_b = 16 + (size_t)rows * K * 4;
  void *ws = nullptr;
  if (cudaMallocAsync(&ws, peak_b + agg_b + flag_b, st) != cudaSuccess) {
    set_error("rave_augment: cudaMallocAsync of %zu bytes failed", peak_b + agg_b + flag_b);
    return 2;
  }
  char *w = static_cast<char *>(ws);
  AugArgs a;
  a.raw = raw;
  a.raw_int16 = raw_int16;
  a.B = B;
  a.C = C;
  a.L = L;
  a.N = N;
  a.K = (int)K;
  a.draws = draws;
  a.key = key;
  a.noise = noise;
  a.out = out;
  a.derivative = derivative;
  a.peak = reinterpret_cast<unsigned long long *>(w);
  a.agg = reinterpret_cast<double *>(w + peak_b);
  a.ticket = reinterpret_cast<unsigned *>(w + peak_b + agg_b);
  a.flag = a.ticket + 4;
  cudaMemsetAsync(a.peak, 0, peak_b, st);
  cudaMemsetAsync(a.ticket, 0, flag_b, st);
  const unsigned grid = (unsigned)(rows * K);
  if (normalize) {
    augment_kernel<1><<<grid, kAugThreads, 0, st>>>(a);
    augment_kernel<2><<<grid, kAugThreads, 0, st>>>(a);
  } else {
    augment_kernel<0><<<grid, kAugThreads, 0, st>>>(a);
  }
  const cudaError_t e = cudaGetLastError();
  cudaFreeAsync(ws, st);
  if (e != cudaSuccess) {
    set_error("rave_augment: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  count_launch(normalize ? 2 : 1);
  return 0;
}
