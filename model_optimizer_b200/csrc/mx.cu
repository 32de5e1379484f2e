// mx.cu -- MX formats: power-of-two (E8M0) scale per block of 8 / 16 / 32 elements.
//
//   fake quant : cuda_ext_mx.fused_amax_convert(inputs, block_size, format, E8M0)
//                kernels/quantization/gemm/tensor_quant_mx.cu:36-54 (quantize), :103-131 (NV E8M0
//                scale), :134-151 (compute_scale), :240-291 (kernel), :320-366 (host entry);
//                element rounding kernels/quantization/gemm/tensor_quant_mx.h:76-190.
//   MXFP8 pack : quantization/qtensor/mxfp8_tensor.py:42-65, 150-262
//   MXFP4 pack : quantization/qtensor/mxfp4_tensor.py:37-144
//
// One thread owns one block: for 16-bit inputs a 32-element block is two 32-byte vectors (four LDG.E.128), the
// block amax is an in-register packed-integer max, the scale is an exponent read off the bits of
// one IEEE division, and because the scale is a power of two the element path is
// mul -> narrow-format rounding (RNE, satfinite) -> back to float -> mul, sign OR-ed back on the
// packed words.  The reference spends one thread per ELEMENT with a cub reduction per block.
//
// Conventions fixed here where the reference leaves them open (its `sign` variable is
// uninitialised for zeros and NaN, tensor_quant_mx.cu:39-43): zeros produce +0.0, NaN elements
// keep sign +.  The reference is built with --use_fast_math; this file follows the source as
// written (IEEE division, no flush-to-zero).
#include <cmath>

#include "block16.cuh"

namespace b200q {

constexpr int kMxThreads = 256;

enum MxFmt { kE4M3 = 0, kE5M2, kINT8, kE0M3, kE1M2, kE3M0, kE2M1, kE3M2, kE2M3, kE8M0 };

__host__ __device__ inline float mx_format_max(int fmt) {  // tensor_quant_mx.h:193-218
  switch (fmt) {
    case kE4M3: return 448.f;
    case kE5M2: return 57344.f;
    case kINT8: return 127.f;
    case kE0M3: return 7.f;
    case kE1M2: return 3.5f;
    case kE3M0: return 16.f;
    case kE2M1: return 6.f;
    case kE3M2: return 28.f;
    case kE2M3: return 7.5f;
    default: return 0.f;
  }
}

// 2^k as fp32 for k in [-149, 127] (denormals included)
__host__ __device__ inline uint32_t pow2_bits(int k) {
  return k >= -126 ? (uint32_t)(k + 127) << 23 : 1u << (k + 149);
}
__device__ __forceinline__ float pow2f(int k) { return __uint_as_float(pow2_bits(k)); }

// exponent of the NV E8M0 scale: unscale = 2^e, scale = 2^-e, e = ceil(log2(fp32(amax / dmax)))
// taken from the bits of the rounded ratio exactly like tensor_quant_mx.cu:112-125
__device__ __forceinline__ int e8m0_exponent_nv(float amax, float dmax) {
  const uint32_t b = __float_as_uint(__fdiv_rn(amax, dmax));
  const int ex = (int)((b >> 23) & 0xffu);
  const uint32_t sig = b & 0x7fffffu;
  const bool up = sig > 0u && ex != 0xfe && !(ex == 0 && sig <= 0x400000u);
  return up ? ex - 126 : ex - 127;
}

// ---- element rounding of non-negative magnitudes (pairs, so the packed FP8 cvt is used) ----
template <int FMT> struct MxRound;

template <> struct MxRound<kE4M3> {
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    e4m3x2_to_f32x2(f32x2_to_e4m3x2(a0, a1), r0, r1);
  }
};
template <> struct MxRound<kE5M2> {
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    uint16_t p;
    uint32_t h2;
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(p) : "f"(a1), "f"(a0));
    asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h2) : "h"(p));
    r0 = h2f_bits((uint16_t)(h2 & 0xffffu));
    r1 = h2f_bits((uint16_t)(h2 >> 16));
  }
};
// the compare chain, not the branch-free e2m1_round_mag of the NVFP4 kernels: in this kernel the branch-free form
// measured slower on an H100 (bf16 [4096, 14336], block 32: 92.5 us with the chain, 100.8 us without)
template <> struct MxRound<kE2M1> {
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = e2m1_round_mag_ref(a0);
    r1 = e2m1_round_mag_ref(a1);
  }
};
template <> struct MxRound<kE3M2> {  // bias 3: minimum normal exponent -2, max 28
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = minifloat_rne_sat<2, -2>(a0, 28.f);
    r1 = minifloat_rne_sat<2, -2>(a1, 28.f);
  }
};
template <> struct MxRound<kE2M3> {  // bias 1: minimum normal exponent 0, max 7.5
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = minifloat_rne_sat<3, 0>(a0, 7.5f);
    r1 = minifloat_rne_sat<3, 0>(a1, 7.5f);
  }
};
template <> struct MxRound<kINT8> {  // rint + clamp (tensor_quant_mx.h:84-93)
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = fminf(rintf(a0), 127.f);
    r1 = fminf(rintf(a1), 127.f);
  }
};
template <> struct MxRound<kE0M3> {  // integers 0..7, ties to even
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = fminf(rintf(a0), 7.f);
    r1 = fminf(rintf(a1), 7.f);
  }
};
template <> struct MxRound<kE1M2> {  // multiples of 0.5 up to 3.5, ties to even
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = fminf(__fmul_rn(rintf(__fmul_rn(a0, 2.f)), 0.5f), 3.5f);
    r1 = fminf(__fmul_rn(rintf(__fmul_rn(a1, 2.f)), 0.5f), 3.5f);
  }
};
template <> struct MxRound<kE3M0> {  // powers of two 0.25 .. 16, ties AWAY from zero (tensor_quant_mx.h:96-104)
  // bounds are 1.5 * 2^k: adding half a binade to the bit pattern and clearing the mantissa rounds
  // m * 2^e (m in [1, 2)) to 2^e for m < 1.5 and to 2^(e+1) from m == 1.5 on; [0.125, 0.375) -> 0.25
  static __device__ __forceinline__ float one(float a) {
    const float p = __uint_as_float((__float_as_uint(a) + 0x00400000u) & 0xff800000u);
    return a < 0.125f ? 0.f : fminf(fmaxf(p, 0.25f), 16.f);
  }
  static __device__ __forceinline__ void pair(float a0, float a1, float &r0, float &r1) {
    r0 = one(a0);
    r1 = one(a1);
  }
};

// non-finite / NaN handling of one magnitude, reference order (tensor_quant_mx.h:122-190):
// E4M3 / E5M2 keep NaN, INT8 maps NaN to 0 (cvt.rni of NaN), table formats saturate NaN and inf
template <int FMT> __device__ __noinline__ float mx_round_slow(float a) {
  if (a != a) {
    if (FMT == kE4M3 || FMT == kE5M2) return a;
    if (FMT == kINT8) return 0.f;
    return mx_format_max(FMT);
  }
  float r0, r1;
  MxRound<FMT>::pair(fminf(a, 3.0e38f), 0.f, r0, r1);
  return r0;
}

// ---------------------------------------------------------------------------------------------
// fake quant, aligned fast path: one thread = one block of NB16*16 elements
// ---------------------------------------------------------------------------------------------
template <typename Tag, int NB16, int FMT> struct MxBlock {
  Block<Tag, 32> b[NB16];

  // careful path (any NaN / inf in the block): reference order, fully unrolled on registers
  __device__ __forceinline__ void careful() {
    constexpr int W = Block<Tag, 32>::WORDS;
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < NB16; ++j) {
#pragma unroll
      for (int i = 0; i < W; ++i) {
        if constexpr (Elem<Tag>::PER_WORD == 2) {
          float lo, hi;
          Elem<Tag>::unpack(b[j].word(i), lo, hi);
          amax = fmaxf(amax, fmaxf(fabsf(lo), fabsf(hi)));  // fmaxf drops NaN (:175-178)
        } else {
          amax = fmaxf(amax, fabsf(__uint_as_float(b[j].word(i))));
        }
      }
    }
    float scale = 1.f, unscale = 1.f;
    if (!(amax == 0.f || amax != amax || amax > 3.4028234664e38f)) {
      const int e = e8m0_exponent_nv(amax, mx_format_max(FMT));
      scale = pow2f(-e);
      unscale = pow2f(e);
    }
    auto one = [&](float v) {
      const float r = __fmul_rn(mx_round_slow<FMT>(__fmul_rn(fabsf(v), scale)), unscale);
      return v < 0.f ? -r : r;
    };
#pragma unroll
    for (int j = 0; j < NB16; ++j) {
#pragma unroll
      for (int i = 0; i < W; ++i) {
        if constexpr (Elem<Tag>::PER_WORD == 2) {
          float lo, hi;
          Elem<Tag>::unpack(b[j].word(i), lo, hi);
          b[j].word(i) = Elem<Tag>::pack(one(lo), one(hi));
        } else {
          b[j].word(i) = __float_as_uint(one(__uint_as_float(b[j].word(i))));
        }
      }
    }
  }

  __device__ __forceinline__ void run() {
    constexpr int W = Block<Tag, 32>::WORDS;
    uint32_t acc = 0;
#pragma unroll
    for (int j = 0; j < NB16; ++j) {
#pragma unroll
      for (int i = 0; i < W; ++i) {
        b[j].word(i) = kill_neg_zero<Tag>(b[j].word(i));
        acc = absmax_acc<Tag>(acc, b[j].word(i));
      }
    }
    const uint32_t mb = Elem<Tag>::absbits_to_f32bits(absmax_collapse<Tag>(acc));
    if (mb >= 0x7f800000u) {
      careful();
      return;
    }
    if (mb == 0u) return;  // all zeros (negative zeros already cleared): out = +0
    const int e = e8m0_exponent_nv(__uint_as_float(mb), mx_format_max(FMT));
    const float scale = pow2f(-e), unscale = pow2f(e);
#pragma unroll
    for (int j = 0; j < NB16; ++j) {
      if constexpr (Elem<Tag>::PER_WORD == 2) {
#pragma unroll
        for (int i = 0; i < W; ++i) {
          const uint32_t w = b[j].word(i);
          float lo, hi, r0, r1;
          Elem<Tag>::unpack(w, lo, hi);
          MxRound<FMT>::pair(__fmul_rn(fabsf(lo), scale), __fmul_rn(fabsf(hi), scale), r0, r1);
          b[j].word(i) = Elem<Tag>::pack(__fmul_rn(r0, unscale), __fmul_rn(r1, unscale)) | (w & Elem<Tag>::NEG_ZERO2);
        }
      } else {
#pragma unroll
        for (int i = 0; i < W; i += 2) {
          const uint32_t w0 = b[j].word(i), w1 = b[j].word(i + 1);
          float r0, r1;
          MxRound<FMT>::pair(__fmul_rn(fabsf(__uint_as_float(w0)), scale),
                             __fmul_rn(fabsf(__uint_as_float(w1)), scale), r0, r1);
          b[j].word(i) = __float_as_uint(__fmul_rn(r0, unscale)) | (w0 & 0x80000000u);
          b[j].word(i + 1) = __float_as_uint(__fmul_rn(r1, unscale)) | (w1 & 0x80000000u);
        }
      }
    }
  }
};

template <typename Tag, int NB16, int FMT>
__global__ void __launch_bounds__(kMxThreads)
    mx_fq_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t n_blocks) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * kMxThreads + threadIdx.x;
  if (i >= n_blocks) return;
  MxBlock<Tag, NB16, FMT> m;
#pragma unroll
  for (int j = 0; j < NB16; ++j) m.b[j].load(x, i * NB16 + j);
  m.run();
#pragma unroll
  for (int j = 0; j < NB16; ++j) m.b[j].store(y, i * NB16 + j);
}

// generic path: block size 8, ragged rows (zero padded tail block, :256-270) or unaligned tensors
template <typename Tag, int FMT>
__global__ void __launch_bounds__(kMxThreads)
    mx_fq_generic_kernel(const void *__restrict__ x, void *__restrict__ y, size_t n_rows, size_t row_len,
                         size_t blocks_per_row, int bs) {
  const size_t total = n_rows * blocks_per_row;
  for (size_t t = blockIdx.x * (size_t)kMxThreads + threadIdx.x; t < total; t += (size_t)gridDim.x * kMxThreads) {
    const size_t row = t / blocks_per_row, c0 = (t % blocks_per_row) * (size_t)bs;
    const int cnt = (int)((row_len - c0) < (size_t)bs ? (row_len - c0) : (size_t)bs);
    const size_t base = row * row_len + c0;
    float amax = 0.f;
    for (int e = 0; e < cnt; ++e) amax = fmaxf(amax, fabsf(Elem<Tag>::load1(x, base + e)));
    float scale = 1.f, unscale = 1.f;
    if (!(amax == 0.f || amax != amax || amax > 3.4028234664e38f)) {
      const int ex = e8m0_exponent_nv(amax, mx_format_max(FMT));
      scale = pow2f(-ex);
      unscale = pow2f(ex);
    }
    for (int e = 0; e < cnt; ++e) {
      const float v = Elem<Tag>::load1(x, base + e);
      const float r = __fmul_rn(mx_round_slow<FMT>(__fmul_rn(fabsf(v), scale)), unscale);
      Elem<Tag>::store1(y, base + e, v < 0.f ? -r : r);
    }
  }
}

template <typename Tag, int FMT>
static int launch_mx_fq(const void *x, void *y, size_t n_rows, size_t row_len, int bs, cudaStream_t st) {
  const size_t n = n_rows * row_len;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), ay = reinterpret_cast<uintptr_t>(y);
  B200Q_REQUIRE(ax % Elem<Tag>::SIZE == 0 && ay % Elem<Tag>::SIZE == 0, "tensor not element-aligned");
  if ((bs == 16 || bs == 32) && row_len % bs == 0 && ax % 32 == 0 && ay % 32 == 0) {
    const size_t n_blocks = n / bs;
    const size_t grid = (n_blocks + kMxThreads - 1) / kMxThreads;
    B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
    const uint8_t *xb = static_cast<const uint8_t *>(x);
    uint8_t *yb = static_cast<uint8_t *>(y);
    if (bs == 32) launch_pdl(mx_fq_kernel<Tag, 2, FMT>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, xb, yb, n_blocks);
    else launch_pdl(mx_fq_kernel<Tag, 1, FMT>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, xb, yb, n_blocks);
    return check_launch("mx_fq_kernel");
  }
  const size_t bpr = (row_len + bs - 1) / bs;
  size_t grid = (n_rows * bpr + kMxThreads - 1) / kMxThreads;
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
  mx_fq_generic_kernel<Tag, FMT><<<(unsigned)grid, kMxThreads, 0, st>>>(x, y, n_rows, row_len, bpr, bs);
  return check_launch("mx_fq_generic_kernel");
}

template <typename Tag>
static int dispatch_mx_fq(const void *x, void *y, size_t n_rows, size_t row_len, int bs, int fmt, cudaStream_t st) {
  switch (fmt) {
    case kE4M3: return launch_mx_fq<Tag, kE4M3>(x, y, n_rows, row_len, bs, st);
    case kE5M2: return launch_mx_fq<Tag, kE5M2>(x, y, n_rows, row_len, bs, st);
    case kINT8: return launch_mx_fq<Tag, kINT8>(x, y, n_rows, row_len, bs, st);
    case kE0M3: return launch_mx_fq<Tag, kE0M3>(x, y, n_rows, row_len, bs, st);
    case kE1M2: return launch_mx_fq<Tag, kE1M2>(x, y, n_rows, row_len, bs, st);
    case kE3M0: return launch_mx_fq<Tag, kE3M0>(x, y, n_rows, row_len, bs, st);
    case kE2M1: return launch_mx_fq<Tag, kE2M1>(x, y, n_rows, row_len, bs, st);
    case kE3M2: return launch_mx_fq<Tag, kE3M2>(x, y, n_rows, row_len, bs, st);
    case kE2M3: return launch_mx_fq<Tag, kE2M3>(x, y, n_rows, row_len, bs, st);
    default: break;
  }
  set_error("unsupported MX element format %d", fmt);
  return B200Q_ERR_INVALID;
}

// ---------------------------------------------------------------------------------------------
// MXFP8 quant-and-pack / unpack (block 32 along the last dim, zero padded)
// ---------------------------------------------------------------------------------------------
// clamp(ceil(log2(r)), -127, 127) for r > 0 else -127 (mxfp8_tensor.py:52-65), exact on the bits
__device__ __forceinline__ int ceil_log2_clamped(float r) {
  if (!(r > 0.f)) return -127;  // zero, negative, NaN
  const uint32_t b = __float_as_uint(r);
  const int ex = (int)(b >> 23);
  if (ex == 0xff) return 127;   // inf
  if (ex == 0) return (b > 0x400000u) ? -126 : -127;  // denormal: only (2^-127, 2^-126) rounds up to -126
  const int e = (ex - 127) + ((b & 0x7fffffu) ? 1 : 0);
  return e > 127 ? 127 : e;
}

// one scaled element to its MXFP8 code: clamp to +-448 (NaN kept), then torch's e4m3fn cast
__device__ __forceinline__ uint8_t mxfp8_cast(float v) {
  if (v == v) v = fminf(fmaxf(v, -448.f), 448.f);
  return f32_to_e4m3fn_torch(v);
}

template <typename Tag>
__global__ void __launch_bounds__(kMxThreads)
    mxfp8_pack_kernel(const void *__restrict__ x, size_t n_rows, size_t row_len, size_t blocks_per_row,
                      const uint8_t *__restrict__ scale_in, uint8_t *__restrict__ q,
                      uint8_t *__restrict__ scale_out, int aligned) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = n_rows * blocks_per_row;
  const size_t t = blockIdx.x * (size_t)kMxThreads + threadIdx.x;
  if (t >= total) return;
  if (aligned) {  // row_len % 32 == 0 and 32-byte aligned pointers: block t is contiguous at element 32 t
    Block<Tag, 32> b[2];
    b[0].load(static_cast<const uint8_t *>(x), 2 * t);
    b[1].load(static_cast<const uint8_t *>(x), 2 * t + 1);
    const uint32_t mb = Elem<Tag>::absbits_to_f32bits(
        max(b[0].absmax_native_bits(), b[1].absmax_native_bits()));
    int byte;
    if (scale_in) byte = scale_in[t];
    else byte = ceil_log2_clamped(__fdiv_rn(__uint_as_float(mb), 448.f)) + 127;
    const float sf = pow2f(127 - byte);
    Vec<32> out;
    const bool finite = mb < 0x7f800000u;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float f[kBlk];
      b[j].to_floats(f);
#pragma unroll
      for (int e = 0; e < kBlk; e += 4) {
        uint32_t w;
        if (finite) {  // satfinite cvt == clamp(+-448) followed by the e4m3fn cast
          w = (uint32_t)f32x2_to_e4m3x2(__fmul_rn(f[e], sf), __fmul_rn(f[e + 1], sf)) |
              ((uint32_t)f32x2_to_e4m3x2(__fmul_rn(f[e + 2], sf), __fmul_rn(f[e + 3], sf)) << 16);
        } else {
          w = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) w |= (uint32_t)mxfp8_cast(__fmul_rn(f[e + k], sf)) << (8 * k);
        }
        out.r[j * 4 + e / 4] = w;
      }
    }
    stg(reinterpret_cast<Vec<32> *>(q) + t, out);
    if (!scale_in) scale_out[t] = (uint8_t)byte;
    return;
  }
  const size_t row = t / blocks_per_row, c0 = (t % blocks_per_row) * 32;
  const int cnt = (int)((row_len - c0) < 32 ? (row_len - c0) : 32);
  const size_t base = row * row_len + c0;
  float amax = 0.f;
  bool nan = false;
  for (int e = 0; e < cnt; ++e) {
    const float a = fabsf(Elem<Tag>::load1(x, base + e));
    nan |= (a != a);
    amax = fmaxf(amax, a);
  }
  if (nan) amax = __uint_as_float(0x7fc00000u);  // torch max propagates NaN
  int byte;
  if (scale_in) byte = scale_in[t];
  else byte = ceil_log2_clamped(__fdiv_rn(amax, 448.f)) + 127;
  const float sf = pow2f(127 - byte);
  for (int e = 0; e < cnt; ++e) q[base + e] = mxfp8_cast(__fmul_rn(Elem<Tag>::load1(x, base + e), sf));
  if (!scale_in) scale_out[t] = (uint8_t)byte;
}

template <typename Tag>
__global__ void __launch_bounds__(kMxThreads)
    mxfp8_unpack_kernel(const uint8_t *__restrict__ q, const uint8_t *__restrict__ scale, size_t n_rows,
                        size_t row_len, size_t blocks_per_row, void *__restrict__ y, int aligned) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = n_rows * blocks_per_row;
  const size_t t = blockIdx.x * (size_t)kMxThreads + threadIdx.x;
  if (t >= total) return;
  const float d = pow2f((int)scale[t] - 127);
  if (aligned) {
    const Vec<32> in = ldg_stream(reinterpret_cast<const Vec<32> *>(q) + t);
    Block<Tag, 32> b[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float f[kBlk];
#pragma unroll
      for (int e = 0; e < kBlk; e += 2) {
        const uint32_t w = in.r[j * 4 + e / 4];
        float lo, hi;
        e4m3x2_to_f32x2((uint16_t)(w >> (16 * ((e / 2) & 1))), lo, hi);
        f[e] = __fmul_rn(lo, d);
        f[e + 1] = __fmul_rn(hi, d);
      }
      b[j].from_floats(f);
      b[j].store(static_cast<uint8_t *>(y), 2 * t + j);
    }
    return;
  }
  const size_t row = t / blocks_per_row, c0 = (t % blocks_per_row) * 32;
  const int cnt = (int)((row_len - c0) < 32 ? (row_len - c0) : 32);
  const size_t base = row * row_len + c0;
  for (int e = 0; e < cnt; ++e) Elem<Tag>::store1(y, base + e, __fmul_rn(e4m3_bits_to_f32(q[base + e]), d));
}

// ---------------------------------------------------------------------------------------------
// MXFP4 quant-and-pack / unpack (flat blocks)
// ---------------------------------------------------------------------------------------------
// code of one scaled value (mxfp4_tensor.py:44-52): sign bit set unless y > 0 (zeros -> 8),
// magnitude = number of E2M1 bounds strictly below |y| (exact ties round down)
__device__ __forceinline__ uint32_t mxfp4_code(float y) {
  const float a = fabsf(y);
  const uint32_t mag = (a > 0.25f) + (a > 0.75f) + (a > 1.25f) + (a > 1.75f) + (a > 2.5f) + (a > 3.5f) + (a > 5.0f);
  return ((y > 0.f) ? 0u : 8u) + mag;
}

template <typename Tag>
__global__ void __launch_bounds__(kMxThreads)
    mxfp4_pack_kernel(const void *__restrict__ x, size_t n_blocks, int bs, uint8_t *__restrict__ q,
                      uint8_t *__restrict__ scale_out, int aligned) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t t = blockIdx.x * (size_t)kMxThreads + threadIdx.x;
  if (t >= n_blocks) return;
  if (aligned) {  // bs == 32, 32-byte aligned input, 16-byte aligned output
    Block<Tag, 32> b[2];
    b[0].load(static_cast<const uint8_t *>(x), 2 * t);
    b[1].load(static_cast<const uint8_t *>(x), 2 * t + 1);
    const uint32_t mb = Elem<Tag>::absbits_to_f32bits(
        max(b[0].absmax_native_bits(), b[1].absmax_native_bits()));
    const float r = __fdiv_rn(__uint_as_float(mb), 6.f);
    int e = -127;
    if (r > 0.f) {
      e = ceil_log2_clamped(r);  // amax / 6 is finite: the upper clamp never binds
      if (__float_as_uint(r) >= 0x7f800000u) e = 128;  // inf amax: exp2(inf) -> x / inf
    }
    const float inv = e >= 128 ? 0.f : pow2f(-e);
    Vec<16> out;
    if constexpr (Elem<Tag>::PER_WORD == 2) {
      // 16-bit inputs: a multiply and an add per element do the scaling and both fix-ups of the reference's rule
      // (mxfp4_tensor.py:44-52: ties round DOWN, sign bit set unless y > 0) on top of the hardware RNE convert:
      //   * x * 2^-e has at most 11 significant bits, so multiplying by 2^-e * (1 - 2^-20) moves every value a few
      //     fp32 ulps towards zero: exact ties fall below their boundary, nothing else crosses one;
      //   * adding -2^-149 (the smallest denormal) to the ROUNDED product turns +0 (and a product that underflowed to
      //     +0) into a negative zero-magnitude value -> code 8 like the reference's zeros, and leaves every other
      //     value's code alone (2^-149 itself becomes +0 -> code 0, as y > 0 demands; normal values absorb it).
      //     One FMA would add it to the exact product instead: a bf16 product in (2^-150, 2^-149), which y rounds up
      //     to 2^-149 > 0, would come out as -0 -> code 8.
      const float inv_t = __fmul_rn(inv, 1.0f - 0x1p-20f);
      const float neg_den = __uint_as_float(0x80000001u);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
#pragma unroll
        for (int i = 0; i < 8; i += 4) {
          uint32_t w = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float lo, hi;
            Elem<Tag>::unpack(b[j].word(i + k), lo, hi);
            w |= f32x2_to_e2m1x2(__fadd_rn(__fmul_rn(lo, inv_t), neg_den), __fadd_rn(__fmul_rn(hi, inv_t), neg_den))
                 << (8 * k);
          }
          out.r[j * 2 + i / 4] = w;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float f[kBlk];
        b[j].to_floats(f);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          uint32_t w = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t c0 = mxfp4_code(__fmul_rn(f[i * 8 + 2 * k], inv));
            const uint32_t c1 = mxfp4_code(__fmul_rn(f[i * 8 + 2 * k + 1], inv));
            w |= (c0 | (c1 << 4)) << (8 * k);
          }
          out.r[j * 2 + i] = w;
        }
      }
    }
    stg(reinterpret_cast<Vec<16> *>(q) + t, out);
    scale_out[t] = (uint8_t)(e + 127);
    return;
  }
  const size_t base = t * (size_t)bs;
  float amax = 0.f;
  for (int e = 0; e < bs; ++e) amax = fmaxf(amax, fabsf(Elem<Tag>::load1(x, base + e)));
  const float r = __fdiv_rn(amax, 6.f);
  int ex = -127;
  if (r > 0.f) {
    ex = ceil_log2_clamped(r);
    if (__float_as_uint(r) >= 0x7f800000u) ex = 128;
  }
  const float inv = ex >= 128 ? 0.f : pow2f(-ex);
  for (int e = 0; e < bs; e += 2) {
    const uint32_t c0 = mxfp4_code(__fmul_rn(Elem<Tag>::load1(x, base + e), inv));
    const uint32_t c1 = mxfp4_code(__fmul_rn(Elem<Tag>::load1(x, base + e + 1), inv));
    q[(base + e) / 2] = (uint8_t)(c0 | (c1 << 4));
  }
  scale_out[t] = (uint8_t)(ex + 127);
}

template <typename Tag>
__global__ void __launch_bounds__(kMxThreads)
    mxfp4_unpack_kernel(const uint8_t *__restrict__ q, const uint8_t *__restrict__ scale, size_t n_blocks,
                        int bs, void *__restrict__ y, int aligned) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t t = blockIdx.x * (size_t)kMxThreads + threadIdx.x;
  if (t >= n_blocks) return;
  const float d = pow2f((int)scale[t] - 127);
  if (aligned) {
    const Vec<16> in = ldg_stream(reinterpret_cast<const Vec<16> *>(q) + t);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float f[kBlk];
#pragma unroll
      for (int e = 0; e < kBlk; e += 2) {
        const uint32_t w = in.r[j * 2 + e / 8];
        const uint32_t h2 = e2m1x2_to_f16x2((w >> (8 * ((e / 2) & 3))) & 0xffu);  // code 8 -> -0.0 (:120-124)
        f[e] = __fmul_rn(h2f_bits((uint16_t)(h2 & 0xffffu)), d);
        f[e + 1] = __fmul_rn(h2f_bits((uint16_t)(h2 >> 16)), d);
      }
      Block<Tag, 32> b;
      b.from_floats(f);
      b.store(static_cast<uint8_t *>(y), 2 * t + j);
    }
    return;
  }
  const size_t base = t * (size_t)bs;
  for (int e = 0; e < bs; e += 2) {
    const uint32_t h2 = e2m1x2_to_f16x2(q[(base + e) / 2]);
    Elem<Tag>::store1(y, base + e, __fmul_rn(h2f_bits((uint16_t)(h2 & 0xffffu)), d));
    Elem<Tag>::store1(y, base + e + 1, __fmul_rn(h2f_bits((uint16_t)(h2 >> 16)), d));
  }
}

// host scalar twin of convert_to_exmy (tensor_quant_mx.cu:399-400): the ext exports a plain function
static float host_e4m3_like(float a, int mbits, int min_exp, float maxv) {
  // RNE onto a grid with `mbits` mantissa bits, subnormal spacing 2^(min_exp - mbits), saturating
  if (a != a) return a;
  if (a >= maxv) return maxv;
  int ex;
  frexpf(a, &ex);  // a = m * 2^ex, m in [0.5, 1)
  int e = ex - 1;
  if (e < min_exp) e = min_exp;
  const float ulp = ldexpf(1.f, e - mbits);
  float r = nearbyintf(a / ulp) * ulp;  // default rounding mode: nearest even
  return r > maxv ? maxv : r;
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_fake_quant_mx(const void *x, void *y, int dtype, size_t n_rows, size_t row_len, int block_size,
                        int elem_format, b200q_stream_t stream) {
  if (n_rows * row_len == 0) return B200Q_OK;
  B200Q_REQUIRE(x != nullptr && y != nullptr, "null pointer");
  B200Q_REQUIRE(block_size == 8 || block_size == 16 || block_size == 32,
                "Blocksize for fused call must be one of {8, 16, 32}");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  B200Q_DISPATCH_DTYPE(dtype, Tag, return dispatch_mx_fq<Tag>(x, y, n_rows, row_len, block_size, elem_format, st));
}

int b200q_pack_mxfp8(const void *x, int dtype, size_t n_rows, size_t row_len, const uint8_t *scale_in,
                     uint8_t *q, uint8_t *scale_out, b200q_stream_t stream) {
  if (n_rows * row_len == 0) return B200Q_OK;
  B200Q_REQUIRE(x != nullptr && q != nullptr && (scale_in != nullptr || scale_out != nullptr), "null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t bpr = (row_len + 31) / 32;
  const size_t grid = (n_rows * bpr + kMxThreads - 1) / kMxThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const int aligned = row_len % 32 == 0 && reinterpret_cast<uintptr_t>(x) % 32 == 0 && reinterpret_cast<uintptr_t>(q) % 32 == 0;
  B200Q_DISPATCH_DTYPE(dtype, Tag, {
    B200Q_REQUIRE(reinterpret_cast<uintptr_t>(x) % Elem<Tag>::SIZE == 0, "x is not element-aligned");
    launch_pdl(mxfp8_pack_kernel<Tag>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, x, n_rows, row_len, bpr,
               scale_in, q, scale_out, aligned);
    return check_launch("mxfp8_pack_kernel");
  });
}

int b200q_unpack_mxfp8(const uint8_t *q, const uint8_t *scale, size_t n_rows, size_t row_len, void *y, int dtype,
                       b200q_stream_t stream) {
  if (n_rows * row_len == 0) return B200Q_OK;
  B200Q_REQUIRE(q != nullptr && scale != nullptr && y != nullptr, "null pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t bpr = (row_len + 31) / 32;
  const size_t grid = (n_rows * bpr + kMxThreads - 1) / kMxThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const int aligned = row_len % 32 == 0 && reinterpret_cast<uintptr_t>(y) % 32 == 0 && reinterpret_cast<uintptr_t>(q) % 32 == 0;
  B200Q_DISPATCH_DTYPE(dtype, Tag, {
    B200Q_REQUIRE(reinterpret_cast<uintptr_t>(y) % Elem<Tag>::SIZE == 0, "y is not element-aligned");
    launch_pdl(mxfp8_unpack_kernel<Tag>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, q, scale, n_rows, row_len,
               bpr, y, aligned);
    return check_launch("mxfp8_unpack_kernel");
  });
}

int b200q_pack_mxfp4(const void *x, int dtype, size_t n_blocks, int block_size, uint8_t *q, uint8_t *scale_out,
                     b200q_stream_t stream) {
  if (n_blocks == 0) return B200Q_OK;
  B200Q_REQUIRE(x != nullptr && q != nullptr && scale_out != nullptr, "null pointer");
  B200Q_REQUIRE(block_size > 0 && block_size % 2 == 0, "block_size must be even");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t grid = (n_blocks + kMxThreads - 1) / kMxThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const int aligned = block_size == 32 && reinterpret_cast<uintptr_t>(x) % 32 == 0 && reinterpret_cast<uintptr_t>(q) % 16 == 0;
  B200Q_DISPATCH_DTYPE(dtype, Tag, {
    B200Q_REQUIRE(reinterpret_cast<uintptr_t>(x) % Elem<Tag>::SIZE == 0, "x is not element-aligned");
    launch_pdl(mxfp4_pack_kernel<Tag>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, x, n_blocks, block_size, q,
               scale_out, aligned);
    return check_launch("mxfp4_pack_kernel");
  });
}

int b200q_unpack_mxfp4(const uint8_t *q, const uint8_t *scale, size_t n_blocks, int block_size, void *y, int dtype,
                       b200q_stream_t stream) {
  if (n_blocks == 0) return B200Q_OK;
  B200Q_REQUIRE(q != nullptr && scale != nullptr && y != nullptr, "null pointer");
  B200Q_REQUIRE(block_size > 0 && block_size % 2 == 0, "block_size must be even");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t grid = (n_blocks + kMxThreads - 1) / kMxThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const int aligned = block_size == 32 && reinterpret_cast<uintptr_t>(y) % 32 == 0 && reinterpret_cast<uintptr_t>(q) % 16 == 0;
  B200Q_DISPATCH_DTYPE(dtype, Tag, {
    B200Q_REQUIRE(reinterpret_cast<uintptr_t>(y) % Elem<Tag>::SIZE == 0, "y is not element-aligned");
    launch_pdl(mxfp4_unpack_kernel<Tag>, dim3((unsigned)grid), dim3(kMxThreads), 0, st, q, scale, n_blocks,
               block_size, y, aligned);
    return check_launch("mxfp4_unpack_kernel");
  });
}

float b200q_convert_to_exmy(float x, int format) {
  const float sign = std::signbit(x) ? -1.f : 1.f;
  const float a = fabsf(x);
  float r;
  switch (format) {
    case kE4M3: r = host_e4m3_like(a, 3, -6, 448.f); break;
    case kE5M2: r = host_e4m3_like(a, 2, -14, 57344.f); break;
    case kINT8: {
      if (a != a) return 0.f;
      r = fminf(nearbyintf(a), 127.f);
      return (x < 0.f && r > 0.f) ? -r : r;  // through an int in the reference: no negative zero
    }
    case kE0M3: r = (a != a) ? 7.f : fminf(nearbyintf(a), 7.f); break;
    case kE1M2: r = (a != a) ? 3.5f : fminf(nearbyintf(a * 2.f) * 0.5f, 3.5f); break;
    case kE3M0:
      r = (a != a) ? 16.f
          : a < 0.125f ? 0.f : a < 0.375f ? 0.25f : a < 0.75f ? 0.5f : a < 1.5f ? 1.f
          : a < 3.f ? 2.f : a < 6.f ? 4.f : a < 12.f ? 8.f : 16.f;
      break;
    case kE2M1: r = (a != a) ? 6.f : host_e4m3_like(a, 1, 0, 6.f); break;
    case kE3M2: r = (a != a) ? 28.f : host_e4m3_like(a, 2, -2, 28.f); break;
    case kE2M3: r = (a != a) ? 7.5f : host_e4m3_like(a, 3, 0, 7.5f); break;
    default: return 0.f;
  }
  if (format != kE4M3 && format != kE5M2 && !(x < 0.f)) return r;  // table formats: sign from `x < 0`
  return sign * r;
}

}  // extern "C"
