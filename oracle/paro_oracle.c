/*
 * paro_oracle.c -- CPU restatement of the ParoQuant hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * call this.  The product path (paroquant_b200/) never links or imports anything under oracle/.
 *
 * What is restated (all citations are into /root/reference):
 *   - AWQ nibble pack / unpack          paroquant/cli/convert.py:19,149-155
 *                                       paroquant/inference/backends/mlx/load.py:15-24
 *   - group dequant  w = (q - z) * s    paroquant/inference/backends/mlx/load.py:46-54 (math),
 *                                       rounded once to the activation dtype T the way the
 *                                       third-party Marlin GEMM forms its operand (SURVEY.md A.3)
 *   - scaled pairwise (Givens) rotation paroquant/kernels/cuda/rotation.cu:10-43,62-95
 *                                       paroquant/kernels/cuda/rotation.cuh:16-75 (fp32),
 *                                       :91-173 (fp16 / bf16 with their rounding points)
 *   - y = xrot . W (+ bias)             paroquant/inference/backends/vllm/plugin.py:281-311
 *                                       paroquant/inference/backends/transformers/modules.py:57-71
 *
 * Parity pin: the reference ships no tests or golden vectors (SURVEY.md section 4), and its kernels
 * are CUDA-only, so they cannot execute in a GPU-less container.  The pin is therefore
 * tests/golden/ref_gpu_*.npz: outputs of the UNMODIFIED reference rotate kernel (compiled by
 * oracle/build_ref.py from the sources where they lie) and of vLLM's Marlin run on an H100 by
 * tools/gen_ref_golden.py.  Until those fixtures exist this oracle is "parity unpinned".
 *
 * One documented deviation: the reference evaluates sin/cos with the GPU's MUFU approximations
 * (__sincosf under --use_fast_math: FMUL.RZ by 1/2pi, MUFU.SIN, MUFU.COS -- seen in the SASS of
 * the reference build).  MUFU tables are not reproducible on a CPU; the oracle uses correctly
 * rounded sinf/cosf.  After the per-stage rounding to T this changes < 1 % of the elements by
 * one ulp of T (measured; tests state the bound).  Everything else (order of operations, single
 * roundings, fmaf contraction c*a + (s*b), flush-to-zero) follows the reference instruction for
 * instruction.
 *
 * dtype codes: 0 = float32, 1 = float16, 2 = bfloat16.  Half types travel as uint16 bit patterns.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PARO_F32 0
#define PARO_F16 1
#define PARO_BF16 2

/* ---------------------------------------------------------------- scalar conversions */

static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* flush-to-zero of fp32 denormals: the reference is built with --use_fast_math (-ftz=true),
 * paroquant/kernels/cuda/__init__.py:30-40; its FMUL/FFMA carry .FTZ in SASS. */
static inline float ftz(float f) {
  uint32_t u = f2u(f);
  if ((u & 0x7f800000u) == 0) u &= 0x80000000u;
  return u2f(u);
}

static inline float bf16_to_f32(uint16_t h) { return u2f((uint32_t)h << 16); }

/* round-to-nearest-even, NaN preserved (matches __float2bfloat16_rn / F2FP.BF16.F32) */
static inline uint16_t f32_to_bf16(float f) {
  uint32_t u = f2u(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x0040u);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

static inline float f16_to_f32(uint16_t h) {
  uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu;
  uint32_t man = h & 0x3ffu;
  if (exp == 0) {
    if (man == 0) return u2f(sign);
    /* subnormal: normalise */
    int e = -1;
    do { man <<= 1; e++; } while (!(man & 0x400u));
    man &= 0x3ffu;
    return u2f(sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13));
  }
  if (exp == 31) return u2f(sign | 0x7f800000u | (man << 13));
  return u2f(sign | ((exp + 112u) << 23) | (man << 13));
}

/* round-to-nearest-even fp32 -> fp16 with subnormal and overflow handling */
static inline uint16_t f32_to_f16(float f) {
  uint32_t u = f2u(f);
  uint32_t sign = (u >> 16) & 0x8000u;
  uint32_t a = u & 0x7fffffffu;
  if (a > 0x7f800000u) return (uint16_t)(sign | 0x7e00u);          /* NaN */
  if (a >= 0x47800000u) {                                           /* >= 65536: inf or overflow */
    return (uint16_t)(sign | 0x7c00u);
  }
  if (a >= 0x38800000u) {                                           /* normal fp16 range */
    uint32_t m = a - 0x38000000u;                                   /* rebias exponent by 112 */
    uint32_t r = m + 0xfffu + ((m >> 13) & 1u);
    return (uint16_t)(sign | (r >> 13));                            /* may carry into inf: correct */
  }
  if (a < 0x33000000u) return (uint16_t)sign;                       /* < 2^-25: rounds to zero */
  /* subnormal result */
  uint32_t e = a >> 23;
  uint32_t m = (a & 0x7fffffu) | 0x800000u;
  uint32_t shift = 126u - e;                                        /* 14 .. 24 */
  uint32_t r = m >> shift;
  uint32_t rem = m & ((1u << shift) - 1u);
  uint32_t half = 1u << (shift - 1u);
  if (rem > half || (rem == half && (r & 1u))) r++;
  return (uint16_t)(sign | r);
}

static inline float half_to_f32(uint16_t h, int dtype) {
  return dtype == PARO_F16 ? f16_to_f32(h) : bf16_to_f32(h);
}
static inline uint16_t f32_to_half(float f, int dtype) {
  return dtype == PARO_F16 ? f32_to_f16(f) : f32_to_bf16(f);
}

/* exported so the python side can validate its numpy conversions against these */
void paro_oracle_f32_to_half(const float *src, uint16_t *dst, int64_t n, int dtype) {
  for (int64_t i = 0; i < n; i++) dst[i] = f32_to_half(src[i], dtype);
}
void paro_oracle_half_to_f32(const uint16_t *src, float *dst, int64_t n, int dtype) {
  for (int64_t i = 0; i < n; i++) dst[i] = half_to_f32(src[i], dtype);
}

/* ---------------------------------------------------------------- AWQ pack / unpack */

/* nibble i (bits 4i..4i+3) of packed[r][c] holds value column 8c + ORDER[i]; convert.py:19 */
static const int AWQ_ORDER[8] = {0, 2, 4, 6, 1, 3, 5, 7};

/* convert.py:149-155 (_pack_awq): values[rows][cols] (0..15) -> packed[rows][cols/8] */
void paro_oracle_awq_pack(const uint8_t *values, int64_t rows, int64_t cols, int32_t *packed) {
  int64_t pc = cols / 8;
  for (int64_t r = 0; r < rows; r++)
    for (int64_t c = 0; c < pc; c++) {
      uint32_t w = 0;
      for (int i = 0; i < 8; i++)
        w |= ((uint32_t)values[r * cols + c * 8 + AWQ_ORDER[i]] & 0xfu) << (4 * i);
      packed[r * pc + c] = (int32_t)w;
    }
}

/* mlx/load.py:21-24 (_unpack_and_reorder): inverse of the above */
void paro_oracle_awq_unpack(const int32_t *packed, int64_t rows, int64_t pcols, uint8_t *values) {
  int64_t cols = pcols * 8;
  for (int64_t r = 0; r < rows; r++)
    for (int64_t c = 0; c < pcols; c++) {
      uint32_t w = (uint32_t)packed[r * pcols + c];
      for (int i = 0; i < 8; i++)
        values[r * cols + c * 8 + AWQ_ORDER[i]] = (uint8_t)((w >> (4 * i)) & 0xfu);
    }
}

/* ---------------------------------------------------------------- dequant
 * W[k][n] = T( (q[k][n] - z[k/G][n]) * s_T[k/G][n] ), returned as fp32 holding a T-representable
 * value.  (q - z) is exact in every T; the product is rounded once (SURVEY.md A.3, confirmed on
 * the H100 against Marlin with one-hot activations, see tests/golden/README.md).
 * For dtype == PARO_F32 the product is the plain fp32 product (mlx/load.py:46-54 math).
 * scales: [K/G][N] as T bit patterns (uint16) for half types, float for f32.            */
void paro_oracle_dequant(const int32_t *qweight, const int32_t *qzeros, const void *scales,
                         int64_t K, int64_t N, int group, int dtype, float *W) {
  int64_t pn = N / 8;
  for (int64_t k = 0; k < K; k++) {
    int64_t g = k / group;
    for (int64_t c = 0; c < pn; c++) {
      uint32_t wq = (uint32_t)qweight[k * pn + c];
      uint32_t wz = (uint32_t)qzeros[g * pn + c];
      for (int i = 0; i < 8; i++) {
        int64_t n = c * 8 + AWQ_ORDER[i];
        int q = (int)((wq >> (4 * i)) & 0xfu);
        int z = (int)((wz >> (4 * i)) & 0xfu);
        float d = (float)(q - z);
        if (dtype == PARO_F32) {
          W[k * N + n] = d * ((const float *)scales)[g * N + n];
        } else {
          float s = half_to_f32(((const uint16_t *)scales)[g * N + n], dtype);
          /* exact fp32 product of two short significands, then ONE rounding to T */
          W[k * N + n] = half_to_f32(f32_to_half(d * s, dtype), dtype);
        }
      }
    }
  }
}

/* ---------------------------------------------------------------- rotation
 * rotation.cu:10-43 + rotation.cuh.  x, out: [M][K] in dtype; idx: [krot][K] int16 local indices;
 * theta: [krot][K/2] ALREADY cast to dtype (rotation.cu:75); scales: [K] already cast to dtype
 * (rotation.cu:76-78) or NULL.  Pairs inside one (r, group) must be disjoint (optim/rotation.py:
 * 33-35 enforces that offline) -- the kernel's result is otherwise a data race; the oracle applies
 * them in thread order t = 0..G/2-1.                                                            */
int paro_oracle_rotate(const void *x, void *out, const int16_t *idx, const void *theta,
                       const void *scales, int64_t M, int64_t K, int krot, int group, int dtype) {
  if (group <= 0 || (group & 1) || K % group != 0) return 1;
  int64_t ngroups = K / group;
  int half = group / 2;
  float *v = (float *)malloc(sizeof(float) * (size_t)group);
  float *sn = (float *)malloc(sizeof(float) * (size_t)krot * (size_t)half);
  float *cs = (float *)malloc(sizeof(float) * (size_t)krot * (size_t)half);
  if (!v || !sn || !cs) { free(v); free(sn); free(cs); return 2; }

  for (int64_t g = 0; g < ngroups; g++) {
    /* load_coeffs (rotation.cuh:35-44,118-129) + __sincosf (:49,136) */
    for (int r = 0; r < krot; r++)
      for (int t = 0; t < half; t++) {
        int64_t ti = (int64_t)r * (K / 2) + g * half + t;
        float th = dtype == PARO_F32 ? ((const float *)theta)[ti]
                                     : half_to_f32(((const uint16_t *)theta)[ti], dtype);
        double thd = (double)th;
        sn[r * half + t] = (float)sin(thd);
        cs[r * half + t] = (float)cos(thd);
      }
    for (int64_t m = 0; m < M; m++) {
      /* load_group: v[c] = T(x * scale) -- one rounding (__hmul), rotation.cuh:110-115;
       * fp32: plain product, rotation.cuh:24-32 */
      for (int c = 0; c < group; c++) {
        int64_t xi = m * K + g * group + c;
        if (dtype == PARO_F32) {
          float xv = ((const float *)x)[xi];
          v[c] = scales ? ftz(ftz(xv) * ftz(((const float *)scales)[g * group + c])) : xv;
        } else {
          float xv = half_to_f32(((const uint16_t *)x)[xi], dtype);
          float sv = scales ? half_to_f32(((const uint16_t *)scales)[g * group + c], dtype) : 1.0f;
          v[c] = half_to_f32(f32_to_half(xv * sv, dtype), dtype);
        }
      }
      /* apply_one x krot, barrier between rotations (rotation.cu:35-39) */
      for (int r = 0; r < krot; r++) {
        const int16_t *p = idx + (int64_t)r * K + g * group;
        for (int t = 0; t < half; t++) {
          int i = p[2 * t], j = p[2 * t + 1];
          if (i < 0 || i >= group || j < 0 || j >= group) { free(v); free(sn); free(cs); return 3; }
          float s_ = sn[r * half + t], c_ = cs[r * half + t];
          float a = ftz(v[i]), b = ftz(v[j]);
          /* SASS of the reference build: FMUL.FTZ p = s*b ; FFMA.FTZ yi = c*a + p ;
           *                              FMUL.FTZ q = s*(-a) ; FFMA.FTZ yj = c*b + q
           * (identical structure for the fp32 instantiation after -fmad contraction). */
          float yi = ftz(fmaf(c_, a, ftz(s_ * b)));
          float yj = ftz(fmaf(c_, b, ftz(s_ * -a)));
          if (dtype == PARO_F32) {
            v[i] = yi; v[j] = yj;
          } else {
            v[i] = half_to_f32(f32_to_half(yi, dtype), dtype);   /* rotation.cuh:152-153 */
            v[j] = half_to_f32(f32_to_half(yj, dtype), dtype);
          }
        }
      }
      for (int c = 0; c < group; c++) {
        int64_t oi = m * K + g * group + c;
        if (dtype == PARO_F32) ((float *)out)[oi] = v[c];
        else ((uint16_t *)out)[oi] = f32_to_half(v[c], dtype);
      }
    }
  }
  free(v); free(sn); free(cs);
  return 0;
}

/* ---------------------------------------------------------------- GEMM
 * y[m][n] = T( sum_k a[m][k] * W[k][n] ) (+ bias in T, plugin.py:309-310).  a: [M][K] in dtype,
 * W: [K][N] fp32 (already T-rounded by paro_oracle_dequant).  Accumulation in double, so the
 * oracle is the "infinitely precise accumulate" reference for any fp32 accumulation order.
 * acc_out (optional, may be NULL): the un-rounded double sums, for error budgets.            */
void paro_oracle_gemm(const void *a, const float *W, const void *bias, int64_t M, int64_t N,
                      int64_t K, int dtype, void *y, double *acc_out) {
  double *acc = (double *)malloc(sizeof(double) * (size_t)N);
  for (int64_t m = 0; m < M; m++) {
    for (int64_t n = 0; n < N; n++) acc[n] = 0.0;
    for (int64_t k = 0; k < K; k++) {
      double av = dtype == PARO_F32 ? (double)((const float *)a)[m * K + k]
                                    : (double)half_to_f32(((const uint16_t *)a)[m * K + k], dtype);
      if (av == 0.0) continue;
      const float *w = W + k * N;
      for (int64_t n = 0; n < N; n++) acc[n] += av * (double)w[n];
    }
    for (int64_t n = 0; n < N; n++) {
      if (acc_out) acc_out[m * N + n] = acc[n];
      if (dtype == PARO_F32) {
        float r = (float)acc[n];
        if (bias) r += ((const float *)bias)[n];
        ((float *)y)[m * N + n] = r;
      } else {
        uint16_t h = f32_to_half((float)acc[n], dtype);
        if (bias) {
          float r = half_to_f32(h, dtype) + half_to_f32(((const uint16_t *)bias)[n], dtype);
          h = f32_to_half(r, dtype);
        }
        ((uint16_t *)y)[m * N + n] = h;
      }
    }
  }
  free(acc);
}

/* ---------------------------------------------------------------- whole linear (n_parts = 1)
 * plugin.py:281-286 / modules.py:57-71: y = rotate(x, pairs, theta, channel_scales) . dequant(W)
 * W (fp32 [K][N]) is passed in so callers dequantise once.                                   */
int paro_oracle_linear(const void *x, const float *W, const int16_t *idx, const void *theta,
                       const void *cscales, const void *bias, int64_t M, int64_t N, int64_t K,
                       int krot, int group, int dtype, void *y, void *xrot_scratch) {
  int rc = paro_oracle_rotate(x, xrot_scratch, idx, theta, cscales, M, K, krot, group, dtype);
  if (rc) return rc;
  paro_oracle_gemm(xrot_scratch, W, bias, M, N, K, dtype, y, NULL);
  return 0;
}
