// intq.cuh -- the integer and FP8-E4M3 per-tensor / per-channel fake-quant rules of one value: the one definition
// that the fake-quant, scale-search, histogram-search, NVFP4 static-scale and GPTQ column kernels share.
#pragma once
#include "common.cuh"

namespace b200q {

// ---------------------------------------------------------------------------------------------
// integer fake quant (tensor_quant_gpu.cu:43-56)
// ---------------------------------------------------------------------------------------------
struct IntQ {
  float scale, y, maxb, minb;
  bool zero, fast;
  // reference order, one element; ref_noinline is apply_vec's rare slow path, kept out of line
  __device__ __forceinline__ static float ref(float x, float s, float hi, float lo) {
    float o = rintf(__fmul_rn(x, s));
    o = o > hi ? hi : o;
    o = o < lo ? lo : o;
    return __fdiv_rn(o, s);
  }
  __device__ __noinline__ static float ref_noinline(float x, float s, float hi, float lo) { return ref(x, s, hi, lo); }
  __device__ __forceinline__ void setup(float amax, float max_bound, float min_bound) {
    maxb = max_bound;
    minb = min_bound;
    zero = amax < (1.0f / (1 << 24));
    scale = __fdiv_rn(max_bound, amax);
    ExactDiv d(scale);
    y = d.y;
    // fast path: hoisted exact division + magic-number RNE (valid while |q| <= 2^21)
    fast = d.ok && scale > 0.f && max_bound <= 2097152.0f;
  }
  // reference order
  __device__ __forceinline__ float apply_ref(float x) const { return zero ? 0.f : ref(x, scale, maxb, minb); }
  // same result as ref when `fast`, branch-free: rint via 1.5*2^23 (round-to-nearest-even of the FADD),
  // NaN-keeping clamps, 3-FFMA exact division; the sign of a zero result comes from x*scale like rint's does
  __device__ __forceinline__ float apply_fast(float x) const {
    const float t = __fmul_rn(x, scale);
    float o = __fadd_rn(__fadd_rn(t, 12582912.0f), -12582912.0f);
    asm("min.NaN.f32 %0, %0, %1;" : "+f"(o) : "f"(maxb));
    asm("max.NaN.f32 %0, %0, %1;" : "+f"(o) : "f"(minb));
    const float q = __fmul_rn(o, y);
    const float r = __fmaf_rn(q, -scale, o);
    return copysignf(__fmaf_rn(y, r, q), t);
  }
  __device__ __forceinline__ float apply(float x) const {
    if (zero) return 0.f;
    return fast ? apply_fast(x) : ref(x, scale, maxb, minb);
  }
  // N elements held in registers: the rare slow path (scale outside the exact-division window, > 21-bit formats)
  // is out of line, still fully unrolled so f[] stays in registers
  template <int N> __device__ __forceinline__ void apply_vec(float *f) const {
    if (zero) {
#pragma unroll
      for (int e = 0; e < N; ++e) f[e] = 0.f;
    } else if (fast) {
#pragma unroll
      for (int e = 0; e < N; ++e) f[e] = apply_fast(f[e]);
    } else {
#pragma unroll
      for (int e = 0; e < N; ++e) f[e] = ref_noinline(f[e], scale, maxb, minb);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// fp8 op
// ---------------------------------------------------------------------------------------------
struct Fp8Scale {
  float scale, inv;
  // eager == false: the CUDA extension's rule, scale = 448.f / amax (IEEE division, tensor_quant_gpu_fp8.cu:94-98)
  // eager == true : _fp8_eager's rule (tensor_quant.py:46-59), where `448.0 / safe_amax` is torch's
  //                 Tensor.__rtruediv__ = safe_amax.reciprocal() * 448.0 (two roundings); used by the reference
  //                 whenever amax has more than one non-singleton dim (2-D block scales) and on CPU
  __device__ __forceinline__ void setup(float amax, bool eager = false) {
    const float safe = (amax <= (1.0f / (1 << 24))) ? 1.0f : amax;
    scale = eager ? __fmul_rn(__frcp_rn(safe), 448.0f) : __fdiv_rn(448.0f, safe);
    inv = __fdiv_rn(1.0f, scale);
  }
  __device__ __forceinline__ float apply(float v) const { return __fmul_rn(e4m3_round(__fmul_rn(v, scale)), inv); }
  // a with this scale and b with sb's, through one packed convert
  __device__ __forceinline__ void apply2(float &a, float &b, const Fp8Scale &sb) const {
    float lo, hi;
    e4m3x2_to_f32x2(f32x2_to_e4m3x2(__fmul_rn(a, scale), __fmul_rn(b, sb.scale)), lo, hi);
    a = __fmul_rn(lo, inv);
    b = __fmul_rn(hi, sb.inv);
  }
  __device__ __forceinline__ void apply2(float &a, float &b) const { apply2(a, b, *this); }
};

}  // namespace b200q
