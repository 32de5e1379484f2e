// intq.cuh -- integer and FP8-E4M3 fake quant of one value (shared by fake_quant.cu, the scale-search kernels and the
// GPTQ column kernel).
#pragma once
#include "common.cuh"

namespace b200q {

// ---------------------------------------------------------------------------------------------
// integer fake quant with the hoisted exact division (same math as fake_quant.cu IntScale)
// ---------------------------------------------------------------------------------------------
struct IntQ {
  float scale, y, maxb, minb;
  bool zero, fast;
  __device__ __forceinline__ void setup(float amax, float max_bound, float min_bound) {
    maxb = max_bound;
    minb = min_bound;
    zero = amax < (1.0f / (1 << 24));
    scale = __fdiv_rn(max_bound, amax);
    ExactDiv d(scale);
    y = d.y;
    fast = d.ok && scale > 0.f && max_bound <= 2097152.0f;
  }
  __device__ __forceinline__ float apply(float x) const {
    if (zero) return 0.f;
    if (fast) {
      const float t = __fmul_rn(x, scale);
      float o = __fadd_rn(__fadd_rn(t, 12582912.0f), -12582912.0f);
      asm("min.NaN.f32 %0, %0, %1;" : "+f"(o) : "f"(maxb));
      asm("max.NaN.f32 %0, %0, %1;" : "+f"(o) : "f"(minb));
      const float q = __fmul_rn(o, y);
      const float r = __fmaf_rn(q, -scale, o);
      return copysignf(__fmaf_rn(y, r, q), t);
    }
    float o = rintf(__fmul_rn(x, scale));
    o = o > maxb ? maxb : o;
    o = o < minb ? minb : o;
    return __fdiv_rn(o, scale);
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
  __device__ __forceinline__ void apply2(float &a, float &b) const {
    float lo, hi;
    e4m3x2_to_f32x2(f32x2_to_e4m3x2(__fmul_rn(a, scale), __fmul_rn(b, scale)), lo, hi);
    a = __fmul_rn(lo, inv);
    b = __fmul_rn(hi, inv);
  }
};

}  // namespace b200q
