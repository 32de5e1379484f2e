// pack.cu -- weight quant-and-pack for INT4 (block-wise "compress" and export layouts) and FP8,
// plus the matching unpack kernels.  HBM-bound: 2 B read + 0.5 / 1 B written per element.
//
// Reference semantics (bit-exact):
//   INT4 compress : quantization/qtensor/int4_tensor.py:52-68 (scales = 7 / amax, i.e.
//                   Tensor.__rtruediv__ = reciprocal() * 7, both rounded to the tensor dtype) +
//                   INT4_quantize_kernel, kernels/quantization/gemm/tensor_quant_gpu.cu:311-340
//                   (all arithmetic in the tensor dtype T, roundf = half away from zero)
//   INT4 unpack   : INT4_dequantize_kernel, tensor_quant_gpu.cu:262-279
//   INT4 export   : pack_int4_in_uint8, export/quant_utils.py:792-833
//   FP8           : FP8QTensor.quantize/dequantize, quantization/qtensor/fp8_tensor.py:41-155;
//                   to_quantized_weight, export/quant_utils.py:854-866
#include "block16.cuh"

namespace b200q {

constexpr int kPkThreads = 256;

template <typename Tag> __device__ __forceinline__ float native_bits_to_float(uint32_t b) {
  return __uint_as_float(Elem<Tag>::absbits_to_f32bits(b));
}

// ---------------------------------------------------------------------------------------------
// INT4 block-wise compress: L lanes (16 elements each) per quant block
// ---------------------------------------------------------------------------------------------
template <typename Tag> __device__ __forceinline__ uint32_t int4_nibble(float x, float s) {
  using E = Elem<Tag>;
  float v = E::round(__fmul_rn(x, s));           // T * T
  v = fmaxf(-8.0f, fminf(7.0f, v));              // max(-(7+1), min(7, v)) on floats: NaN -> 7
  const float u = E::round(__fadd_rn(v, 8.0f));  // T + T, 0 <= u <= 15
  if constexpr (E::SIZE == 2) {
    // roundf(u), 0 <= u <= 15 on the 16-bit grid, without the XU-pipe F2I: nudging u by 2^-13 (less
    // than half the grid spacing next to any k + 0.5 tie) turns "half away from zero" into plain
    // round-to-nearest, which the 2^23 magic-number add performs; the integer sits in the low mantissa bits
    return __float_as_uint(__fadd_rn(__fadd_rn(u, 0x1p-13f), 8388608.0f)) & 0xFu;
  } else {
    return (uint32_t)((int)roundf(u)) & 0xFu;
  }
}

// 16-bit tensors: the reference kernel's arithmetic is T arithmetic (tensor_quant_gpu.cu:311-340), so the PACKED
// hardware ops on a word of two elements give the same bits as the per-element emulation above at half the
// instructions: mul.rn / min / max / add.rn on bf16x2 (f16x2) -- the product of two 8-bit (11-bit) significands is
// exact before its single rounding, min / max return the non-NaN operand like fminf / fmaxf, and v + 8 is exact in
// fp32 whenever it is not absorbed.  Only the final round-half-away-from-zero runs per element in fp32: one FMA
// u * (1 + 2^-13) + 2^23 -- the relative nudge is below T's relative spacing, so only exact k + 0.5 ties move (up).
// (Packed16<Tag>: common.cuh)
// one word (elements e, e + 1) -> the byte first << 4 | second
template <typename Tag> __device__ __forceinline__ uint32_t int4_byte_packed(uint32_t w, uint32_t s2) {
  using P = Packed16<Tag>;
  uint32_t v = P::mul(w, s2);
  v = P::mx(P::NEG_EIGHT, P::mn(P::SEVEN, v));
  const uint32_t u2 = P::add(v, P::EIGHT);
  float u0, u1;
  Elem<Tag>::unpack(u2, u0, u1);
  const uint32_t n0 = __float_as_uint(__fmaf_rn(u0, 1.0f + 0x1p-13f, 8388608.0f));
  const uint32_t n1 = __float_as_uint(__fmaf_rn(u1, 1.0f + 0x1p-13f, 8388608.0f));
  return ((n0 & 0xFu) << 4) | (n1 & 0xFu);
}

template <typename Tag, int VB, int L>
__global__ void __launch_bounds__(kPkThreads)
    int4_pack_kernel(const uint8_t *__restrict__ x, size_t n_chunks, uint8_t *__restrict__ scales_out,
                     uint2 *__restrict__ packed) {
  using E = Elem<Tag>;
  constexpr int U = 2;  // two 16-element chunks per thread (kPkThreads apart: lane groups stay aligned)
  pdl_launch_dependents();
  pdl_wait();
  const size_t base = (size_t)blockIdx.x * (kPkThreads * U) + threadIdx.x;
  Block<Tag, VB> b[U];
  uint32_t m[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const size_t i = base + (size_t)u * kPkThreads;
    m[u] = 0;
    if (i < n_chunks) b[u].load(x, i);
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const size_t i = base + (size_t)u * kPkThreads;
    if (i < n_chunks) m[u] = b[u].absmax_native_bits();
    m[u] = group_max<L>(m[u]);  // quant-block amax (exact in T)
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const size_t i = base + (size_t)u * kPkThreads;
    if (i >= n_chunks) continue;
    // scales = 7 / amax == amax.reciprocal() * 7, each step rounded to T (torch Tensor.__rtruediv__)
    const float amax = native_bits_to_float<Tag>(m[u]);
    const float r = E::round(__fdiv_rn(1.0f, amax));
    const float s = E::round(__fmul_rn(r, 7.0f));
    if ((threadIdx.x & (L - 1)) == 0) {
      const size_t blk = i / L;
      if constexpr (E::SIZE == 2) {
        uint16_t bits;
        if constexpr (std::is_same<Tag, BF16Tag>::value) bits = f2bf_bits(s);
        else bits = f2h_bits(s);
        reinterpret_cast<uint16_t *>(scales_out)[blk] = bits;
      } else {
        reinterpret_cast<float *>(scales_out)[blk] = s;
      }
    }
    uint32_t lo = 0, hi = 0;
    if constexpr (E::SIZE == 2) {
      const uint32_t sb = Packed16<Tag>::bits(s), s2 = sb | (sb << 16);
#pragma unroll
      for (int e = 0; e < kBlk; e += 2) {
        const uint32_t byte = int4_byte_packed<Tag>(b[u].word(e / 2), s2);
        if (e < 8) lo |= byte << (4 * e);
        else hi |= byte << (4 * (e - 8));
      }
    } else {
      float f[kBlk];
      b[u].to_floats(f);
#pragma unroll
      for (int e = 0; e < kBlk; e += 2) {
        // byte = first << 4 | second ; bytes are laid out little-endian in the 8-byte store
        const uint32_t byte = (int4_nibble<Tag>(f[e], s) << 4) | int4_nibble<Tag>(f[e + 1], s);
        if (e < 8) lo |= byte << (4 * e);
        else hi |= byte << (4 * (e - 8));
      }
    }
    packed[i] = make_uint2(lo, hi);
  }
}

// generic: one thread per quant block, scalar I/O (block sizes that are not 16 * 2^k, odd alignment)
template <typename Tag>
__global__ void __launch_bounds__(kPkThreads)
    int4_pack_generic_kernel(const void *__restrict__ x, size_t n_blocks, int block_size,
                             void *__restrict__ scales_out, uint8_t *__restrict__ packed) {
  using E = Elem<Tag>;
  const size_t b = (size_t)blockIdx.x * kPkThreads + threadIdx.x;
  if (b >= n_blocks) return;
  const size_t base = b * (size_t)block_size;
  float amax = 0.f;
  bool nan = false;
  for (int e = 0; e < block_size; ++e) {
    const float a = fabsf(E::load1(x, base + e));
    if (a != a) nan = true;
    amax = fmaxf(amax, a);
  }
  if (nan) amax = __uint_as_float(0x7fc00000u);
  const float r = E::round(__fdiv_rn(1.0f, amax));
  const float s = E::round(__fmul_rn(r, 7.0f));
  E::store1(scales_out, b, s);
  for (int e = 0; e < block_size; e += 2) {
    const uint32_t byte = (int4_nibble<Tag>(E::load1(x, base + e), s) << 4) |
                          int4_nibble<Tag>(E::load1(x, base + e + 1), s);
    packed[(base + e) / 2] = (uint8_t)byte;
  }
}

template <typename Tag>
static int launch_int4_pack(const void *x, size_t n, int block_size, void *scales_out,
                            uint8_t *packed, cudaStream_t st) {
  if (n == 0) return B200Q_OK;
  B200Q_REQUIRE(block_size >= 2 && block_size % 2 == 0 && n % (size_t)block_size == 0,
                "n must be a multiple of an even block_size");
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x);
  const int L = block_size / kBlk;
  const bool pow2 = block_size % kBlk == 0 && (L & (L - 1)) == 0 && L <= 32;
  if (pow2 && ax % 16 == 0 && reinterpret_cast<uintptr_t>(packed) % 8 == 0) {
    const size_t n_chunks = n / kBlk;
    const size_t grid = (n_chunks + 2 * kPkThreads - 1) / (2 * kPkThreads);
    B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
    const uint8_t *xb = static_cast<const uint8_t *>(x);
    uint8_t *sc = static_cast<uint8_t *>(scales_out);
    uint2 *pk = reinterpret_cast<uint2 *>(packed);
    const bool v32 = ax % 32 == 0;
#define LAUNCH(VB_, L_) launch_pdl(int4_pack_kernel<Tag, VB_, L_>, dim3((unsigned)grid), dim3(kPkThreads), 0, st, xb, n_chunks, sc, pk)
#define LAUNCH_L(VB_)                                                                              \
  switch (L) {                                                                                     \
  case 1: LAUNCH(VB_, 1); break;                                                                   \
  case 2: LAUNCH(VB_, 2); break;                                                                   \
  case 4: LAUNCH(VB_, 4); break;                                                                   \
  case 8: LAUNCH(VB_, 8); break;                                                                   \
  case 16: LAUNCH(VB_, 16); break;                                                                 \
  default: LAUNCH(VB_, 32); break;                                                                 \
  }
    if (v32) { LAUNCH_L(32) } else { LAUNCH_L(16) }
#undef LAUNCH_L
#undef LAUNCH
    return check_launch("int4_pack_kernel");
  }
  const size_t n_blocks = n / (size_t)block_size;
  const size_t grid = (n_blocks + kPkThreads - 1) / kPkThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  int4_pack_generic_kernel<Tag><<<(unsigned)grid, kPkThreads, 0, st>>>(x, n_blocks, block_size, scales_out, packed);
  return check_launch("int4_pack_generic_kernel");
}

// unpack: one thread per packed byte pair group of 8 bytes (16 elements)
template <typename Tag>
__global__ void __launch_bounds__(kPkThreads)
    int4_unpack_kernel(const uint8_t *__restrict__ packed, const void *__restrict__ scales, size_t n,
                       int block_size, void *__restrict__ y) {
  using E = Elem<Tag>;
  for (size_t byte = (size_t)blockIdx.x * kPkThreads + threadIdx.x; byte < n / 2;
       byte += (size_t)gridDim.x * kPkThreads) {
    const uint32_t p = packed[byte];
    const float s = E::load1(scales, (byte * 2) / (size_t)block_size);
    const float a = (float)((int)(p >> 4) - 8), b = (float)((int)(p & 0xFu) - 8);
    E::store1(y, 2 * byte, __fdiv_rn(a, s));
    E::store1(y, 2 * byte + 1, __fdiv_rn(b, s));
  }
}

// ---------------------------------------------------------------------------------------------
// INT4 export pack: pairs consecutive OUTPUT channels; one thread = EPV columns x 2 rows
// ---------------------------------------------------------------------------------------------
template <typename Tag, int RES /*0: f32, 1: bf16, 2: f16*/>
__global__ void __launch_bounds__(kPkThreads)
    int4_export_kernel(const void *__restrict__ w, size_t out_dim, size_t in_dim,
                       const void *__restrict__ scale, int scale_dtype, int block_size,
                       uint8_t *__restrict__ packed) {
  using E = Elem<Tag>;
  const size_t total = (out_dim / 2) * in_dim;
  const size_t nsb = in_dim / (size_t)block_size;
  for (size_t t = (size_t)blockIdx.x * kPkThreads + threadIdx.x; t < total;
       t += (size_t)gridDim.x * kPkThreads) {
    const size_t op = t / in_dim, i = t % in_dim;
    uint32_t q[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const size_t o = 2 * op + k;
      const float s = load_scalar(scale, scale_dtype, o * nsb + i / (size_t)block_size);
      float v = __fdiv_rn(E::load1(w, o * in_dim + i), s);
      if constexpr (RES == 1) v = Elem<BF16Tag>::round(v);
      if constexpr (RES == 2) v = Elem<F16Tag>::round(v);
      v = rintf(v);
      v = fminf(fmaxf(v, -8.0f), 7.0f);  // torch.clamp; NaN -> to(int8) is 0 on CUDA / CPU alike
      const int qi = (v != v) ? 0 : (int)v;
      q[k] = (uint32_t)qi & 0xFu;
    }
    packed[t] = (uint8_t)(q[0] | (q[1] << 4));
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 pack / unpack
// ---------------------------------------------------------------------------------------------
// two floats -> two torch-style e4m3fn bytes (RNE; |v| > 464 or NaN -> 0x7f | sign), lo in bits 0..7
__device__ __forceinline__ uint32_t f32x2_to_e4m3fn_torch(float a, float b) {
  uint32_t r = f32x2_to_e4m3x2(a, b);
  if (!(fabsf(a) <= 464.0f)) r = (r & 0xff00u) | 0x7fu | ((__float_as_uint(a) >> 24) & 0x80u);
  if (!(fabsf(b) <= 464.0f)) r = (r & 0x00ffu) | ((0x7fu | ((__float_as_uint(b) >> 24) & 0x80u)) << 8);
  return r;
}

__device__ __noinline__ float fp8_div_noinline(float a, float b) { return __fdiv_rn(a, b); }

// INT8 codes (INT8QTensor.quantize, qtensor/int8_tensor.py:36-86): (x / scale).round().clamp(-128, 127).to(int8) --
// the same division, then round-half-even in T and a clamp; NaN -> 0 (what the CUDA cast makes of it)
__device__ __forceinline__ uint32_t int8_code(float r) {
  float v = rintf(r);
  v = fminf(fmaxf(v, -128.0f), 127.0f);           // NaN -> -128 here, replaced below
  return (r != r) ? 0u : ((uint32_t)(int)v & 0xffu);
}

template <typename Tag, int VB, bool ROUND_TO_T, bool INT8>
__global__ void __launch_bounds__(kPkThreads)
    fp8_pack_kernel(const uint8_t *__restrict__ x, size_t nvec, const void *__restrict__ scale,
                    int scale_dtype, size_t n_scale, size_t outer, uint8_t *__restrict__ q) {
  using E = Elem<Tag>;
  constexpr int EPV = VB / E::SIZE;
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * kPkThreads + threadIdx.x;
  if (i >= nvec) return;
  const Vec<VB> v = ldg_stream(reinterpret_cast<const Vec<VB> *>(x) + i);
  float f[EPV];
  vec_to_floats<Tag, VB>(v, f);
  uint32_t out[EPV / 4];
  const bool uniform = (n_scale == 1) || (outer % EPV == 0);
  float s0 = 1.f;
  if (uniform) s0 = load_scalar(scale, scale_dtype, n_scale == 1 ? 0 : ((i * EPV) / outer) % n_scale);
  const ExactDiv d(s0);
  // vector-level |x| max on the raw words decides the path once per 16 elements: the hoisted exact
  // division is valid for |x| <= 2^60 (tiny operands only ever round to a zero code, whose sign
  // copysign restores) and the torch-cast overflow rule (|q| > 464 -> NaN) cannot fire when
  // max|x| <= 448 * s (quotient rounding adds < 1 %).  Otherwise: plain div.rn + per-element checks.
  uint32_t mbits = 0;
#pragma unroll
  for (int w = 0; w < Vec<VB>::WORDS; ++w) mbits = absmax_acc<Tag>(mbits, v.r[w]);
  const float vmax = __uint_as_float(E::absbits_to_f32bits(absmax_collapse<Tag>(mbits)));
  const bool fast = uniform && d.ok && s0 > 0.f && vmax <= 0x1p60f && (INT8 || vmax <= __fmul_rn(448.0f, s0));
  if (fast) {
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      float r = copysignf(d.quot(f[e]), f[e]);
      if constexpr (ROUND_TO_T) r = E::round(r);
      f[e] = r;
    }
#pragma unroll
    for (int k = 0; k < EPV / 4; ++k) {
      if constexpr (INT8) {
        // finite quotients: magic-number round-half-even (|q| <= 2^22 after the clamp) instead of rintf + F2I
        uint32_t w = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float c = fminf(fmaxf(f[4 * k + j], -128.0f), 127.0f);
          w |= (__float_as_uint(__fadd_rn(c, 12582912.0f)) & 0xffu) << (8 * j);
        }
        out[k] = w;
      } else {
        out[k] = (uint32_t)f32x2_to_e4m3x2(f[4 * k], f[4 * k + 1]) | ((uint32_t)f32x2_to_e4m3x2(f[4 * k + 2], f[4 * k + 3]) << 16);
      }
    }
  } else {
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      const float sc = uniform ? s0 : load_scalar(scale, scale_dtype, ((i * EPV + e) / outer) % n_scale);
      float r = fp8_div_noinline(f[e], sc);
      if constexpr (ROUND_TO_T) r = E::round(r);
      f[e] = r;
    }
#pragma unroll
    for (int k = 0; k < EPV / 4; ++k) {
      if constexpr (INT8)
        out[k] = int8_code(f[4 * k]) | (int8_code(f[4 * k + 1]) << 8) | (int8_code(f[4 * k + 2]) << 16) | (int8_code(f[4 * k + 3]) << 24);
      else
        out[k] = f32x2_to_e4m3fn_torch(f[4 * k], f[4 * k + 1]) | (f32x2_to_e4m3fn_torch(f[4 * k + 2], f[4 * k + 3]) << 16);
    }
  }
  uint32_t *dst = reinterpret_cast<uint32_t *>(q + i * EPV);
#pragma unroll
  for (int k = 0; k < EPV / 4; ++k) dst[k] = out[k];
}

template <typename Tag, bool ROUND_TO_T, bool INT8>
__global__ void __launch_bounds__(kPkThreads)
    fp8_pack_scalar_kernel(const void *__restrict__ x, size_t begin, size_t end,
                           const void *__restrict__ scale, int scale_dtype, size_t n_scale,
                           size_t outer, uint8_t *__restrict__ q) {
  using E = Elem<Tag>;
  for (size_t i = begin + (size_t)blockIdx.x * kPkThreads + threadIdx.x; i < end;
       i += (size_t)gridDim.x * kPkThreads) {
    float r = __fdiv_rn(E::load1(x, i), load_scalar(scale, scale_dtype, n_scale == 1 ? 0 : (i / outer) % n_scale));
    if constexpr (ROUND_TO_T) r = E::round(r);
    if constexpr (INT8) q[i] = (uint8_t)int8_code(r);
    else q[i] = f32_to_e4m3fn_torch(r);
  }
}

template <typename Tag, bool INT8>
__global__ void __launch_bounds__(kPkThreads)
    fp8_unpack_kernel(const uint8_t *__restrict__ q, const void *__restrict__ scale, int scale_dtype,
                      size_t n_scale, size_t outer, void *__restrict__ y, size_t n) {
  using E = Elem<Tag>;
  for (size_t i = (size_t)blockIdx.x * kPkThreads + threadIdx.x; i < n;
       i += (size_t)gridDim.x * kPkThreads) {
    // quantized_data.to(dtype) * scales.to(dtype), computed in dtype (fp8_tensor.py:155)
    const float v = INT8 ? (float)(int8_t)q[i] : E::round(e4m3_bits_to_f32(q[i]));   // int8 values are exact in T
    const float s = E::round(load_scalar(scale, scale_dtype, n_scale == 1 ? 0 : (i / outer) % n_scale));
    E::store1(y, i, __fmul_rn(v, s));
  }
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_pack_int4_blockwise(const void *x, int dtype, size_t n, int block_size, void *scales_out,
                              uint8_t *packed, b200q_stream_t stream) {
  B200Q_REQUIRE((x != nullptr && scales_out != nullptr && packed != nullptr) || n == 0, "null pointer");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_int4_pack<Tag>(x, n, block_size, scales_out, packed, (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_unpack_int4_blockwise(const uint8_t *packed, const void *scales, int dtype, size_t n,
                                int block_size, void *y, b200q_stream_t stream) {
  if (n == 0) return B200Q_OK;
  B200Q_REQUIRE(packed != nullptr && scales != nullptr && y != nullptr, "null pointer");
  B200Q_REQUIRE(block_size >= 2 && n % 2 == 0, "bad block_size / n");
  size_t grid = (n / 2 + kPkThreads - 1) / kPkThreads;
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       int4_unpack_kernel<Tag><<<(unsigned)grid, kPkThreads, 0, (cudaStream_t)stream>>>(
                           packed, scales, n, block_size, y));
  return check_launch("int4_unpack_kernel");
}

int b200q_pack_int4_export(const void *w, int dtype, size_t out_dim, size_t in_dim,
                           const void *scale, int scale_dtype, int block_size, uint8_t *packed,
                           b200q_stream_t stream) {
  if (out_dim * in_dim == 0) return B200Q_OK;
  B200Q_REQUIRE(w != nullptr && scale != nullptr && packed != nullptr, "null pointer");
  B200Q_REQUIRE(out_dim % 2 == 0, "Cannot pack weight. Out dimension %zu is not an even number.", out_dim);
  B200Q_REQUIRE(block_size >= 1 && in_dim % (size_t)block_size == 0, "in_dim must be a multiple of block_size");
  B200Q_REQUIRE(dtype_ok(scale_dtype), "bad scale dtype");
  size_t grid = ((out_dim / 2) * in_dim + kPkThreads - 1) / kPkThreads;
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
  // torch type promotion of w / scale: same dtype keeps it, anything else lands on float32
  const int res = (dtype == scale_dtype) ? (dtype == B200Q_BF16 ? 1 : dtype == B200Q_F16 ? 2 : 0) : 0;
#define LAUNCH(RES_)                                                                               \
  int4_export_kernel<Tag, RES_><<<(unsigned)grid, kPkThreads, 0, (cudaStream_t)stream>>>(          \
      w, out_dim, in_dim, scale, scale_dtype, block_size, packed)
  B200Q_DISPATCH_DTYPE(dtype, Tag, if (res == 1) LAUNCH(1); else if (res == 2) LAUNCH(2); else LAUNCH(0));
#undef LAUNCH
  return check_launch("int4_export_kernel");
}

static int pack_byte_codes(const void *x, int dtype, size_t n, const void *scale, int scale_dtype,
                           size_t n_scale, size_t outer, uint8_t *q, b200q_stream_t stream, bool int8) {
  if (n == 0) return B200Q_OK;
  B200Q_REQUIRE(x != nullptr && scale != nullptr && q != nullptr, "null pointer");
  B200Q_REQUIRE(dtype_ok(scale_dtype) && n_scale >= 1 && outer >= 1, "bad scale arguments");
  // result dtype of x / scale in torch: x's dtype if the scale has it too or is a 0-dim fp32
  // tensor (n_scale == 1), otherwise float32 (no intermediate rounding)
  const bool round_t = (dtype != B200Q_F32) && (scale_dtype == dtype || n_scale == 1);
  cudaStream_t st = (cudaStream_t)stream;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), aq = reinterpret_cast<uintptr_t>(q);
  size_t done = 0;
  if (ax % 16 == 0 && aq % 4 == 0) {
    const bool v32 = ax % 32 == 0;
    const size_t epv = (v32 ? 32 : 16) / dtype_size(dtype);
    const size_t nvec = n / epv;
    if (nvec > 0) {
      const size_t grid = (nvec + kPkThreads - 1) / kPkThreads;
      B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
      const uint8_t *xb = static_cast<const uint8_t *>(x);
#define LAUNCH(VB_, R_, I_) launch_pdl(fp8_pack_kernel<Tag, VB_, R_, I_>, dim3((unsigned)grid), dim3(kPkThreads), 0, st, xb, nvec, scale, scale_dtype, n_scale, outer, q)
#define LAUNCH_I(VB_, R_) do { if (int8) LAUNCH(VB_, R_, true); else LAUNCH(VB_, R_, false); } while (0)
      B200Q_DISPATCH_DTYPE(dtype, Tag, if (v32) { if (round_t) LAUNCH_I(32, true); else LAUNCH_I(32, false); } else { if (round_t) LAUNCH_I(16, true); else LAUNCH_I(16, false); });
#undef LAUNCH_I
#undef LAUNCH
      int rc = check_launch("fp8_pack_kernel");
      if (rc != B200Q_OK) return rc;
      done = nvec * epv;
    }
  }
  if (done < n) {
    size_t grid = (n - done + kPkThreads - 1) / kPkThreads;
    const size_t cap = (size_t)sm_count() * 32;
    if (grid > cap) grid = cap;
#define LAUNCH(R_, I_) fp8_pack_scalar_kernel<Tag, R_, I_><<<(unsigned)grid, kPkThreads, 0, st>>>(x, done, n, scale, scale_dtype, n_scale, outer, q)
#define LAUNCH_I(R_) do { if (int8) LAUNCH(R_, true); else LAUNCH(R_, false); } while (0)
    B200Q_DISPATCH_DTYPE(dtype, Tag, if (round_t) LAUNCH_I(true); else LAUNCH_I(false));
#undef LAUNCH_I
#undef LAUNCH
    return check_launch("fp8_pack_scalar_kernel");
  }
  return B200Q_OK;
}

static int unpack_byte_codes(const uint8_t *q, const void *scale, int scale_dtype, size_t n_scale,
                             size_t outer, void *y, int dtype, size_t n, b200q_stream_t stream, bool int8) {
  if (n == 0) return B200Q_OK;
  B200Q_REQUIRE(q != nullptr && scale != nullptr && y != nullptr, "null pointer");
  B200Q_REQUIRE(dtype_ok(scale_dtype) && n_scale >= 1 && outer >= 1, "bad scale arguments");
  size_t grid = (n + kPkThreads - 1) / kPkThreads;
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
#define LAUNCH(I_) fp8_unpack_kernel<Tag, I_><<<(unsigned)grid, kPkThreads, 0, (cudaStream_t)stream>>>(q, scale, scale_dtype, n_scale, outer, y, n)
  B200Q_DISPATCH_DTYPE(dtype, Tag, if (int8) LAUNCH(true); else LAUNCH(false));
#undef LAUNCH
  return check_launch("fp8_unpack_kernel");
}

int b200q_pack_fp8(const void *x, int dtype, size_t n, const void *scale, int scale_dtype,
                   size_t n_scale, size_t outer, uint8_t *q, b200q_stream_t stream) {
  return pack_byte_codes(x, dtype, n, scale, scale_dtype, n_scale, outer, q, stream, false);
}
int b200q_unpack_fp8(const uint8_t *q, const void *scale, int scale_dtype, size_t n_scale,
                     size_t outer, void *y, int dtype, size_t n, b200q_stream_t stream) {
  return unpack_byte_codes(q, scale, scale_dtype, n_scale, outer, y, dtype, n, stream, false);
}
int b200q_pack_int8(const void *x, int dtype, size_t n, const void *scale, int scale_dtype,
                    size_t n_scale, size_t outer, int8_t *q, b200q_stream_t stream) {
  return pack_byte_codes(x, dtype, n, scale, scale_dtype, n_scale, outer, reinterpret_cast<uint8_t *>(q), stream, true);
}
int b200q_unpack_int8(const int8_t *q, const void *scale, int scale_dtype, size_t n_scale,
                      size_t outer, void *y, int dtype, size_t n, b200q_stream_t stream) {
  return unpack_byte_codes(reinterpret_cast<const uint8_t *>(q), scale, scale_dtype, n_scale, outer, y, dtype, n, stream, true);
}

}  // extern "C"
