// histogram.cu -- histogram collect for HistogramCalibrator: ONE pass over the activation
// (2 B/element) instead of the reference's abs() / float() / max() / histc chain
// (quantization/calib/histogram.py:77-130).
//
// Bin placement restates ATen's CUDA histc (aten/src/ATen/native/cuda/SummaryOps.cu, getBin):
//   bin = (int)((v - min) * nbins / (max - min)) in fp32 with min = 0, bin == nbins -> nbins - 1,
//   elements outside [min, max] (and NaN) are skipped.  The division by the (tensor-uniform) range
//   uses the hoisted exact division, so the bin index is bit-identical to an IEEE divide.
//   Two ranges where that formula has no usable value (DESIGN.md section 4, "Histogram ranges"): a zero range
//   (max = 0) counts its zeros in bin nbins / 2 and skips every other value, and a product v * nbins that overflows
//   fp32 (max above FLT_MAX / nbins) lands in the last bin.  Both only reach the exact-division fallback.
// Counts are privatised per CTA in shared memory (u32 atomics) and flushed once with float
// atomicAdd (histc returns float counts; integer-valued floats add exactly below 2^24).
#include <cuda_fp16.h>
#include <type_traits>

#include "block16.cuh"

namespace b200q {

constexpr int kHistThreads = 512;          // block_log2_hist_kernel
// histogram_kernel, two layouts of the CTA-private counters (knob "hist_variant"):
//   single copy  : one u32 counter per bin (bins < kHsBins), 512 threads, several CTAs per SM
//   lane private : 32 u16 copies of bins < kHcPriv, lane L only ever touches bank L (no bank conflicts), 1024 threads
constexpr int kHsBins = 8192;
constexpr int kHcPriv = 2048;
constexpr size_t kHcSmem = (size_t)kHcPriv * 32 * sizeof(uint16_t);   // 128 KB
constexpr size_t kHcMaxElemsPerCta = 2000000;   // a u16 lane counter sees <= elems / 32 increments

// Device-resident histogram plan (b200q_hist_plan): what HistogramCalibrator.collect decides on the host in
// the reference (calib/histogram.py:111-130) -- first batch: range [0, x_max], width = linspace step; later
// batches: if x_max exceeds the upper edge, nbins = ceil(x_max / width) and the upper edge becomes the last entry
// of arange(0, x_max + width, width).  Kept on the device so that collect never synchronises.
struct HistPlan {
  float upper;       // histc max (= calib_bin_edges[-1])
  float width;       // bin width fixed by the first batch
  float xmax_grow;   // x_max of the batch that last grew the range (to rebuild the edges on the host)
  int nbins;         // current number of bins
  int initialized;
  int overflow;      // 1: a batch needed more than `capacity` bins; 2: a zero-width range had to grow.  Either way
                     // the histogram is no longer the reference's, and later batches are not counted
  int n_growths;
  int reserved;
};

__global__ void hist_plan_kernel(const float *__restrict__ batch_amax, int nbins0, int capacity,
                                 HistPlan *__restrict__ st) {
  const float xmax = batch_amax[0];
  if (!st->initialized) {
    st->upper = xmax;
    st->width = __fdiv_rn(xmax, (float)nbins0);          // torch.linspace(0, x_max, n + 1)[1]
    st->xmax_grow = xmax;
    st->nbins = nbins0;
    st->initialized = 1;
    st->overflow = 0;
    st->n_growths = 0;
    return;
  }
  if (xmax > st->upper) {                                 // histogram.py:121
    const float width = st->width;
    if (!(width > 0.0f)) {                                // an all-zero first batch: a zero-width range cannot grow
      st->overflow = 2;
      return;
    }
    // int((x_max / width).ceil().item()).  Until the first growth the reference's edges come from linspace on the host,
    // so width is a CPU scalar, and torch divides a device tensor by a CPU scalar as x_max * (1 / width); from then on
    // its edges are a device arange and the division is a true one.
    const float quot = st->n_growths == 0 ? __fmul_rn(xmax, __frcp_rn(width)) : __fdiv_rn(xmax, width);
    const int nb = (int)ceilf(quot);
    if (nb > capacity || !(nb > 0)) {
      st->overflow = 1;
      return;
    }
    const float end = __fadd_rn(xmax, width);             // torch.arange(0, x_max + width, width)
    const long long size = (long long)ceil((double)end / (double)width);
    st->upper = (float)((double)(size - 1) * (double)width);
    st->nbins = nb;
    st->xmax_grow = xmax;
    st->n_growths += 1;
  }
}

// bin = trunc(v * nbins / vmax) with the hoisted exact division and an RZ add instead of F2I; the count goes to the
// CTA-private shared counters (fire-and-forget RED.shared), the tail of a grown range to global atomics.
__device__ __noinline__ void hist_cold_add(float *p) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(1.0f) : "memory");
}

template <bool FAST, bool LANEPRIV>
__device__ __forceinline__ void hist_put(float v, float vmax, float fbins, float y, int last, uint32_t sbase,
                                         float *__restrict__ hist) {
  const bool valid = (v >= 0.0f) && (v <= vmax);          // NaN and out-of-range values are skipped (histc)
  const float t = __fmul_rn(v, fbins);
  float q;
  if constexpr (FAST) {
    const float p = __fmul_rn(t, y);
    q = __fmaf_rn(y, __fmaf_rn(p, -vmax, t), p);
  } else {
    // a zero range counts its zeros in bin nbins / 2, as histc widens [0, 0] to [-1, 1]; a product v * nbins that
    // overflows fp32 saturates to the last bin instead of wrapping to bin 0 (inf & 0x7fffff == 0)
    q = vmax > 0.0f ? fminf(__fdiv_rn(t, vmax), fbins) : 0.5f * fbins;
  }
  int bin = (int)(__float_as_uint(__fadd_rz(q, 8388608.0f)) & 0x7fffffu);   // trunc(q), 0 <= q < 2^23
  bin = min(bin, last);
  if (valid) {
    if (__builtin_expect(bin < (LANEPRIV ? kHcPriv : kHsBins), 1)) {
      if constexpr (LANEPRIV) {
        const uint32_t addr = sbase + (((uint32_t)bin & ~1u) << 6);         // word (bin >> 1) * 32 + lane
        const uint32_t one = (bin & 1) ? 0x10000u : 1u;
        asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(addr), "r"(one) : "memory");
      } else {
        asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(sbase + ((uint32_t)bin << 2)), "r"(1u) : "memory");
      }
    } else {
      hist_cold_add(hist + bin);
    }
  }
}

template <typename Tag, int VB, bool FAST, bool LANEPRIV, int THREADS>
__device__ __forceinline__ void hist_stream(const uint8_t *__restrict__ x, size_t head, size_t nvec, size_t tail,
                                            int take_abs, float vmax, float fbins, float y, int last,
                                            uint32_t sbase, float *__restrict__ hist) {
  constexpr int EPV = VB / Elem<Tag>::SIZE;
  const Vec<VB> *xv = reinterpret_cast<const Vec<VB> *>(x + head * Elem<Tag>::SIZE);
  const uint32_t absmask = take_abs ? Elem<Tag>::ABS_MASK : 0xffffffffu;
  auto eat = [&](Vec<VB> v) {
#pragma unroll
    for (int w = 0; w < Vec<VB>::WORDS; ++w) v.r[w] &= absmask;              // |x| on the packed words
    float f[EPV];
    vec_to_floats<Tag, VB>(v, f);
#pragma unroll
    for (int e = 0; e < EPV; ++e) hist_put<FAST, LANEPRIV>(f[e], vmax, fbins, y, last, sbase, hist);
  };
  const size_t stride = (size_t)gridDim.x * THREADS;
  size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  for (; i + stride < nvec; i += 2 * stride) {                               // two loads in flight per thread
    const Vec<VB> a = ldg_stream(xv + i);
    const Vec<VB> b = ldg_stream(xv + i + stride);
    eat(a);
    eat(b);
  }
  if (i < nvec) eat(ldg_stream(xv + i));
  if (blockIdx.x == 0) {
    for (size_t k = threadIdx.x; k < head + tail; k += THREADS) {
      const size_t e = k < head ? k : (head + nvec * EPV + (k - head));
      float v = Elem<Tag>::load1(x, e);
      if (take_abs) v = fabsf(v);
      hist_put<FAST, LANEPRIV>(v, vmax, fbins, y, last, sbase, hist);
    }
  }
}

template <typename Tag, int VB, bool LANEPRIV, int THREADS>
__global__ void __launch_bounds__(THREADS)
    histogram_kernel(const uint8_t *__restrict__ x, size_t head, size_t nvec, size_t tail,
                     int take_abs, const float *__restrict__ range_max, int nbins_arg,
                     const HistPlan *__restrict__ plan, float *__restrict__ hist) {
  extern __shared__ uint32_t s_cnt[];
  const int nbins = plan ? plan->nbins : nbins_arg;
  const float vmax = plan ? plan->upper : range_max[0];
  if (plan && plan->overflow) return;
  const int npriv = min(nbins, LANEPRIV ? kHcPriv : kHsBins);
  const int nwords = LANEPRIV ? ((npriv + 1) >> 1) * 32 : npriv;
  for (int w = threadIdx.x; w < nwords; w += THREADS) s_cnt[w] = 0u;
  __syncthreads();
  const float fbins = (float)nbins;
  const ExactDiv d(vmax);
  // the hoisted exact division holds for every in-range value when the range is ordinary: products
  // below the window only ever land in bin 0 (their quotient is < 1)
  const bool fast = d.ok && vmax > 0.f && __fmul_rn(vmax, fbins) <= 0x1p60f;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(s_cnt) + (LANEPRIV ? lane * 4u : 0u);
  const int last = nbins - 1;
  if (fast) hist_stream<Tag, VB, true, LANEPRIV, THREADS>(x, head, nvec, tail, take_abs, vmax, fbins, d.y, last, sbase, hist);
  else hist_stream<Tag, VB, false, LANEPRIV, THREADS>(x, head, nvec, tail, take_abs, vmax, fbins, d.y, last, sbase, hist);
  __syncthreads();
  if constexpr (LANEPRIV) {
    // flush: a warp sums the 32 lane copies of a bin pair (one word per lane, conflict-free) by shuffles
    const int warp = threadIdx.x >> 5;
    for (int w = warp; w < (npriv + 1) >> 1; w += THREADS / 32) {
      const uint32_t c = s_cnt[w * 32 + lane];
      uint32_t lo = c & 0xffffu, hi = c >> 16;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        lo += __shfl_xor_sync(0xffffffffu, lo, o);
        hi += __shfl_xor_sync(0xffffffffu, hi, o);
      }
      if (lane == 0 && lo) atomicAdd(&hist[2 * w], (float)lo);
      if (lane == 1 && hi) atomicAdd(&hist[2 * w + 1], (float)hi);
    }
  } else {
    for (int b2 = threadIdx.x; b2 < npriv; b2 += THREADS) {
      const uint32_t c = s_cnt[b2];
      if (c) atomicAdd(&hist[b2], (float)c);
    }
  }
}

// ---- 16-bit inputs: count VALUE PATTERNS, bin afterwards ---------------------------------------------------------
// A bf16 / fp16 magnitude has only 2^15 patterns, and histc's bin is a function of the value alone.  So the streaming
// pass does no floating-point work at all: it counts the 15-bit |x| patterns in a CTA-private u32[32768] table
// (3.5 instructions and one RED.shared per element instead of ~23 instructions), flushes the non-zero counters to a
// global u32[32768] scratch, and a 32768-thread epilogue kernel evaluates the exact bin formula ONCE per pattern
// (IEEE division, the formula the element-wise kernel reproduces), adds the counts and clears the scratch.
constexpr int kPatThreads = 1024;
constexpr int kPatterns = 32768;

// Generic form (fp16, and bf16 with knob hist_hot=0): one CTA-private u32[32768] table.  32 random addresses cost ~3.4
// shared-memory wavefronts per warp instruction (bank conflicts), and RED.shared retires about one wavefront per 2.3
// cycles per SM -- that, not HBM, bounds this form.
template <typename Tag>
__global__ void __launch_bounds__(kPatThreads, 1)
    hist_pattern_count_kernel(const uint8_t *__restrict__ x, size_t head, size_t nvec, size_t tail,
                              uint32_t *__restrict__ scratch) {
  static_assert(Elem<Tag>::SIZE == 2, "pattern counting is for 16-bit element types");
  extern __shared__ uint32_t s_pat[];                       // [32768]
  pdl_launch_dependents();
  for (int w = threadIdx.x; w < kPatterns; w += kPatThreads) s_pat[w] = 0u;
  pdl_wait();
  __syncthreads();
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(s_pat);
  auto count_word = [&](uint32_t w) {
    const uint32_t a0 = sbase + ((w & 0x7fffu) << 2), a1 = sbase + ((w >> 14) & 0x1fffcu);   // (w >> 16 & 0x7fff) * 4
    asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a0), "r"(1u) : "memory");
    asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a1), "r"(1u) : "memory");
  };
  using V = Vec<32>;
  const size_t nv32 = nvec / 2;                             // nvec counts 16-byte vectors; the body uses 32-byte loads
  const bool al32 = (reinterpret_cast<uintptr_t>(x + head * 2) % 32) == 0;
  const size_t stride = (size_t)gridDim.x * kPatThreads;
  if (al32) {
    const V *xv = reinterpret_cast<const V *>(x + head * 2);
    size_t i = (size_t)blockIdx.x * kPatThreads + threadIdx.x;
    for (; i + stride < nv32; i += 2 * stride) {            // two 32-byte loads in flight per thread
      const V a = ldg_stream(xv + i);
      const V b = ldg_stream(xv + i + stride);
#pragma unroll
      for (int w = 0; w < V::WORDS; ++w) count_word(a.r[w]);
#pragma unroll
      for (int w = 0; w < V::WORDS; ++w) count_word(b.r[w]);
    }
    if (i < nv32) {
      const V a = ldg_stream(xv + i);
#pragma unroll
      for (int w = 0; w < V::WORDS; ++w) count_word(a.r[w]);
    }
  } else {
    const Vec<16> *xv = reinterpret_cast<const Vec<16> *>(x + head * 2);
    for (size_t i = (size_t)blockIdx.x * kPatThreads + threadIdx.x; i < nv32 * 2; i += stride) {
      const Vec<16> a = ldg_stream(xv + i);
#pragma unroll
      for (int w = 0; w < Vec<16>::WORDS; ++w) count_word(a.r[w]);
    }
  }
  if (blockIdx.x == 0) {                                    // ragged ends + an odd trailing 16-byte vector
    const size_t body = nv32 * 2 * 8;                       // elements covered above
    const size_t rest = head + (nvec * 8 - body) + tail;
    for (size_t k = threadIdx.x; k < rest; k += kPatThreads) {
      const size_t e = k < head ? k : (head + body + (k - head));
      const uint32_t m = reinterpret_cast<const uint16_t *>(x)[e] & 0x7fffu;
      asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(sbase + (m << 2)), "r"(1u) : "memory");
    }
  }
  __syncthreads();
  // flush; every CTA starts at a different pattern so that the CTAs do not walk the same global counters in lock step
  const int start = (int)((blockIdx.x * 2053u) & (kPatterns - 1));
  for (int k = threadIdx.x; k < kPatterns; k += kPatThreads) {
    const int w = (start + k) & (kPatterns - 1);
    const uint32_t c = s_pat[w];
    if (c) atomicAdd(scratch + w, c);
  }
}

// bf16 form: a LANE-PRIVATE hot window.  bf16 has 128 patterns per binade, so the kHot = 1536 patterns under the top
// of the range span 12 binades (values down to upper / 4096): counter (d, lane) lives in word d * 32 + lane, lane L only
// ever touches bank L, and every RED.shared is ONE wavefront.  What falls outside the window is rare for activations:
//   * below the window, when nbins <= 4000, the value is < upper / 4096 and lands in bin 0 whatever it is (q < 1): it is
//     counted in a register and credited to pattern 0 -- this also takes exact zeros (padding, ReLU) off the atomics;
//   * otherwise (huge nbins, or a pattern above the range / NaN, which histc skips) it goes to the global scratch
//     with its exact pattern.
// The main loop is branch-free per element (mask, subtract, clamp, address, RED, running max of d); the
// out-of-window elements of a 32-byte vector are revisited only when that running max says there are any.
constexpr int kHot = 1536;
constexpr size_t kHotSmem = (size_t)(kHot + 1) * 32 * sizeof(uint32_t);    // 192 KB + the dump row

__global__ void __launch_bounds__(kPatThreads, 1)
    hist_pattern_hot_kernel(const uint8_t *__restrict__ x, size_t head, size_t nvec, size_t tail,
                            const float *__restrict__ range_max, int nbins_arg, const HistPlan *__restrict__ plan,
                            uint32_t *__restrict__ scratch) {
  extern __shared__ uint32_t s_pat[];                       // [kHot + 1][32]
  __shared__ uint32_t s_low;
  pdl_launch_dependents();                                  // the bin kernel may queue up behind this grid
  {
    uint4 *z = reinterpret_cast<uint4 *>(s_pat);
    for (int w = threadIdx.x; w < (kHot + 1) * 32 / 4; w += kPatThreads) z[w] = make_uint4(0u, 0u, 0u, 0u);
    if (threadIdx.x == 0) s_low = 0u;
  }
  pdl_wait();                                               // the plan / range of the previous kernel is read below
  __syncthreads();
  const float vmax = plan ? plan->upper : range_max[0];
  const int nbins = plan ? plan->nbins : nbins_arg;
  uint32_t top = __float_as_uint(vmax) >> 16;               // the largest bf16 pattern whose value is <= upper
  top = (vmax >= 0.f && top < 0x7fffu) ? top : 0x7fffu;
  const bool low_is_bin0 = nbins <= 4000;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t hot_base = (uint32_t)__cvta_generic_to_shared(s_pat) + lane * 4u;
  uint32_t low = 0;
  // an element outside the window.  Patterns above `top` (values above the range, NaN) are skipped: histc ignores them
  auto count_slow = [&](uint32_t m) {
    if (m > top) return;
    if (m == 0u) ++low;
    else atomicAdd(scratch + m, 1u);
  };
  auto count_fast = [&](uint32_t m, uint32_t &dmax) {
    const uint32_t d = top - m;                             // wraps to a huge value for m > top
    // no predicate, no branch: out-of-window elements bump a dump row (index kHot) that nobody reads
    // (increment as the literal 1: ptxas then emits ATOMS.POPC.INC, which retires ~2x faster than a register ATOMS.ADD)
    asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(hot_base + (min(d, (uint32_t)kHot) << 7)));
    dmax = max(dmax, d);
  };
  const uint32_t span = top - (uint32_t)kHot;               // below-window patterns are d in [kHot, top]  (top >= kHot)
  auto count_vec = [&](const uint32_t *r, int words) {
    uint32_t dmax = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      if (w < words) {
        count_fast(r[w] & 0x7fffu, dmax);
        count_fast((r[w] >> 16) & 0x7fffu, dmax);
      }
    }
    if (dmax >= (uint32_t)kHot && top >= (uint32_t)kHot) {
      uint32_t top2 = top;
      asm volatile("" : "+r"(top2));                        // keeps the window tests below out of the main loop's CSE
      if (low_is_bin0) {                                    // branch-free: count the elements below the window
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          if (w < words) {
            const uint32_t m0 = r[w] & 0x7fffu, m1 = (r[w] >> 16) & 0x7fffu;
            low += (top2 - m0 - (uint32_t)kHot <= span) ? 1u : 0u;
            low += (top2 - m1 - (uint32_t)kHot <= span) ? 1u : 0u;
          }
        }
      } else {
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          if (w < words) {
            const uint32_t m0 = r[w] & 0x7fffu, m1 = (r[w] >> 16) & 0x7fffu;
            if (top2 - m0 >= (uint32_t)kHot) count_slow(m0);
            if (top2 - m1 >= (uint32_t)kHot) count_slow(m1);
          }
        }
      }
    }
  };
  using V = Vec<32>;
  const size_t nv32 = nvec / 2;                             // nvec counts 16-byte vectors; the body uses 32-byte loads
  const bool al32 = (reinterpret_cast<uintptr_t>(x + head * 2) % 32) == 0;
  const size_t stride = (size_t)gridDim.x * kPatThreads;
  if (al32) {
    const V *xv = reinterpret_cast<const V *>(x + head * 2);
    size_t i = (size_t)blockIdx.x * kPatThreads + threadIdx.x;
    for (; i + stride < nv32; i += 2 * stride) {            // two 32-byte loads in flight per thread
      const V a = ldg_stream(xv + i);
      const V b = ldg_stream(xv + i + stride);
      count_vec(a.r, V::WORDS);
      count_vec(b.r, V::WORDS);
    }
    if (i < nv32) {
      const V a = ldg_stream(xv + i);
      count_vec(a.r, V::WORDS);
    }
  } else {
    const Vec<16> *xv = reinterpret_cast<const Vec<16> *>(x + head * 2);
    for (size_t i = (size_t)blockIdx.x * kPatThreads + threadIdx.x; i < nv32 * 2; i += stride) {
      const Vec<16> a = ldg_stream(xv + i);
      count_vec(a.r, Vec<16>::WORDS);
    }
  }
  if (blockIdx.x == 0) {                                    // ragged ends + an odd trailing 16-byte vector
    const size_t body = nv32 * 2 * 8;                       // elements covered above
    const size_t rest = head + (nvec * 8 - body) + tail;
    for (size_t k = threadIdx.x; k < rest; k += kPatThreads) {
      const size_t e = k < head ? k : (head + body + (k - head));
      const uint32_t m = reinterpret_cast<const uint16_t *>(x)[e] & 0x7fffu;
      uint32_t dmax = 0;
      count_fast(m, dmax);
      if (dmax >= (uint32_t)kHot && m <= top) {
        if (low_is_bin0) ++low;
        else count_slow(m);
      }
    }
  }
  low = __reduce_add_sync(0xffffffffu, low);
  if (lane == 0 && low) atomicAdd(&s_low, low);
  __syncthreads();
  if (threadIdx.x == 0 && s_low) atomicAdd(scratch, s_low);  // credited to pattern 0 (value 0 -> bin 0)
  // flush: thread t sums the 32 lane copies of patterns t, t + 1024 (rotated 16-byte reads: conflict-free) and STORES the
  // totals into this CTA's own row of the global scratch -- no atomics; the bin kernel adds the rows up.  (The first
  // version flushed with one global atomic per (CTA, pattern): 132 CTAs hammering the same 1536 addresses in the same
  // order took 60 % of the kernel.)
  uint32_t *row = scratch + kPatterns + (size_t)blockIdx.x * kHot;
  for (int d = threadIdx.x; d < kHot; d += kPatThreads) {
    const uint4 *q = reinterpret_cast<const uint4 *>(s_pat + d * 32);
    uint32_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {                           // 8 x LDS.128; a quarter-warp covers all 32 banks once
      const uint4 v = q[(j + threadIdx.x) & 7];
      c += (v.x + v.y) + (v.z + v.w);
    }
    row[d] = c;
  }
}

template <typename Tag>
__global__ void __launch_bounds__(kPatThreads)
    hist_pattern_bin_kernel(uint32_t *__restrict__ scratch, const float *__restrict__ range_max, int nbins_arg,
                            const HistPlan *__restrict__ plan, float *__restrict__ hist, int n_hot_rows) {
  const int g = blockIdx.x * kPatThreads + threadIdx.x;    // grid = kPatterns / kPatThreads CTAs exactly
  pdl_wait();                                               // launched programmatically behind the counting grid
  const bool overflow = plan && plan->overflow;
  const int nbins = plan ? plan->nbins : nbins_arg;
  const float vmax = plan ? plan->upper : range_max[0];
  auto add = [&](uint32_t m, uint32_t c) {                  // the exact histc bin of pattern m, once per pattern
    const float v = __uint_as_float(Elem<Tag>::absbits_to_f32bits(m));
    if (overflow || !(v >= 0.0f && v <= vmax)) return;      // NaN patterns and values above the range are skipped (histc)
    const float fbins = (float)nbins;                       // zero range and overflowing product: as in hist_put
    const float q = vmax > 0.0f ? fminf(__fdiv_rn(__fmul_rn(v, fbins), vmax), fbins) : 0.5f * fbins;
    int bin = (int)(__float_as_uint(__fadd_rz(q, 8388608.0f)) & 0x7fffffu);
    bin = min(bin, nbins - 1);
    atomicAdd(hist + bin, (float)c);
  };
  const uint32_t c = scratch[g];                            // table form / out-of-window patterns (atomic counters)
  if (c != 0u) {
    scratch[g] = 0u;                                        // ready for the next batch
    add((uint32_t)g, c);
  }
  if (n_hot_rows > 0) {
    // per-CTA rows of the hot window.  CTA b owns patterns d in [48 b, 48 b + 48); 21 threads per pattern each add up
    // every 21st row (coalesced 192-byte reads), the partials meet in shared memory, and ONE atomic per pattern goes
    // to the histogram (atomics per (part, pattern) serialise on the few low bins: 20 us instead of 3).
    constexpr int kPer = kHot / (kPatterns / kPatThreads);  // 48 patterns per CTA
    constexpr int kParts = kPatThreads / kPer;              // 21 parts (16 threads idle)
    __shared__ uint32_t s_part[kParts][kPer];
    const int dd = threadIdx.x % kPer, part = threadIdx.x / kPer;
    const int d = blockIdx.x * kPer + dd;
    if (part < kParts) {
      const uint32_t *rows = scratch + kPatterns;
      uint32_t sum = 0;
      for (int r = part; r < n_hot_rows; r += kParts) sum += rows[(size_t)r * kHot + d];
      s_part[part][dd] = sum;
    }
    __syncthreads();
    if (threadIdx.x < kPer) {
      uint32_t sum = 0;
#pragma unroll
      for (int k = 0; k < kParts; ++k) sum += s_part[k][threadIdx.x];
      uint32_t top = __float_as_uint(vmax) >> 16;           // as in hist_pattern_hot_kernel
      top = (vmax >= 0.f && top < 0x7fffu) ? top : 0x7fffu;
      if (sum != 0u && (uint32_t)d <= top) add(top - (uint32_t)d, sum);
    }
  }
}

template <typename Tag>
static int launch_histogram(const void *x, size_t n, int take_abs, const float *range_max,
                            int nbins, const HistPlan *plan, float *hist, uint32_t *scratch, cudaStream_t st) {
  if (n == 0) return B200Q_OK;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
  B200Q_REQUIRE(addr % Elem<Tag>::SIZE == 0, "x is not element-aligned");
  constexpr int VB = 16;
  size_t head = ((size_t)VB - addr % VB) % VB / Elem<Tag>::SIZE;
  if (head > n) head = n;
  const size_t epv = VB / Elem<Tag>::SIZE;
  const size_t nvec = (n - head) / epv;
  const size_t tail = n - head - nvec * epv;
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  if constexpr (Elem<Tag>::SIZE == 2) {
    if (scratch != nullptr && take_abs && tuning("hist_variant", 3) == 3) {
      size_t grid = (nvec / 2 + kPatThreads - 1) / kPatThreads;
      const size_t cap = (size_t)sm_count();
      if (grid > cap) grid = cap;
      if (grid == 0) grid = 1;
      bool hot = false;
      if constexpr (std::is_same<Tag, BF16Tag>::value) hot = tuning("hist_hot", 1) == 1;
      if (grid > (size_t)B200Q_HIST_HOT_ROWS) grid = B200Q_HIST_HOT_ROWS;   // scratch holds that many per-CTA rows
      if (hot) {
        auto kern = hist_pattern_hot_kernel;
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHotSmem);
        launch_pdl(kern, dim3((unsigned)grid), dim3(kPatThreads), kHotSmem, st, xb, head, nvec, tail, range_max, nbins, plan,
                   scratch);
      } else {
        const size_t smem = (size_t)kPatterns * sizeof(uint32_t);
        auto kern = hist_pattern_count_kernel<Tag>;
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        launch_pdl(kern, dim3((unsigned)grid), dim3(kPatThreads), smem, st, xb, head, nvec, tail, scratch);
      }
      launch_pdl(hist_pattern_bin_kernel<Tag>, dim3(kPatterns / kPatThreads), dim3(kPatThreads), 0, st, scratch, range_max,
                 nbins, plan, hist, hot ? (int)grid : 0);
      return check_launch("hist_pattern_count_kernel");
    }
  }
  const bool lane_private = tuning("hist_variant", 2) == 1;
  if (lane_private) {
    constexpr int T = 1024;
    size_t grid = (nvec + T - 1) / T;
    const size_t cap = (size_t)sm_count() * (size_t)tuning("hist_ctas_per_sm", 1);
    if (grid > cap) grid = cap;
    const size_t need = (n + kHcMaxElemsPerCta - 1) / kHcMaxElemsPerCta;   // u16 counters: bound a CTA's share
    if (grid < need) grid = need;
    if (grid == 0) grid = 1;
    B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
    auto kern = histogram_kernel<Tag, VB, true, T>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHcSmem);
    kern<<<(unsigned)grid, T, kHcSmem, st>>>(xb, head, nvec, tail, take_abs, range_max, nbins, plan, hist);
  } else {
    constexpr int T = 512;
    size_t grid = (nvec + T - 1) / T;
    const size_t cap = (size_t)sm_count() * (size_t)tuning("hist_ctas_per_sm", 2);
    if (grid > cap) grid = cap;
    if (grid == 0) grid = 1;
    // the planned path sizes the counters for the common (ungrown) range; an explicit nbins uses what it needs
    const int nsm = plan ? kHsBins : (nbins < kHsBins ? nbins : kHsBins);
    const size_t smem = (size_t)nsm * sizeof(uint32_t);
    auto kern = histogram_kernel<Tag, VB, false, T>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<(unsigned)grid, T, smem, st>>>(xb, head, nvec, tail, take_abs, range_max, nbins, plan, hist);
  }
  return check_launch("histogram_kernel");
}

// ---------------------------------------------------------------------------------------------
// NVFP4 activation headroom: log2 histogram of per-block amax (calib/nvfp4_act_headroom.py:110-149)
// ---------------------------------------------------------------------------------------------
// One tensor (descs == nullptr): a grid-stride loop over its n_blocks blocks into hist / max_slot.  A table of tensors
// (descs: MultiDesc, unit = 16-element block, first_cta counted in tiles of kHistThreads = 512 blocks, as
// ops.TensorTable builds it; n_blocks = the table's tile count): CTA c takes tiles 2c and 2c + 1, each found by binary
// search and counted in a shared-memory histogram of its own, so every thread has two block loads in flight; tile t's
// counts / running max go to row slot_t of hist ([n_slots][nbins]) and max_slot[slot_t], and entries sharing a slot
// accumulate.  Both launches bin through the same code, so the grouped launch bins every block exactly as the
// per-tensor one does.
constexpr int kHistTilesPerCta = 2;

template <typename Tag, int VB>
__global__ void __launch_bounds__(kHistThreads)
    block_log2_hist_kernel(const uint8_t *__restrict__ x, size_t n_blocks, const MultiDesc *__restrict__ descs,
                           int n_desc, float log2_min, float range, int nbins, unsigned long long *__restrict__ hist,
                           uint32_t *__restrict__ max_slot) {
  extern __shared__ uint32_t s_hist[];                    // [1 or kHistTilesPerCta][nbins]
  const int n_hist = descs != nullptr ? kHistTilesPerCta : 1;
  for (int b = threadIdx.x; b < n_hist * nbins; b += kHistThreads) s_hist[b] = 0u;
  const float fbins = (float)nbins;
  // bins block b into the histogram h; returns its amax as fp32 bits
  auto bin_block = [&](Block<Tag, VB> &b, uint32_t *h) -> uint32_t {
    const uint32_t fb = Elem<Tag>::absbits_to_f32bits(b.absmax_native_bits());
    const float v = __uint_as_float(fb);
    if (v > 0.0f) {  // NaN fails the test and only shows up in the running max
      const float frac = __fdiv_rn(__fsub_rn(log2f(v), log2_min), range);
      long long idx = (long long)floorf(__fmul_rn(frac, fbins));
      idx = idx < 0 ? 0 : (idx > nbins - 1 ? nbins - 1 : idx);
      atomicAdd(&h[(int)idx], 1u);
    }
    return fb;
  };
  if (descs != nullptr) {
    const size_t t0 = (size_t)blockIdx.x * kHistTilesPerCta;
    Block<Tag, VB> blk[kHistTilesPerCta];
    long long slot[kHistTilesPerCta];
    bool have[kHistTilesPerCta];                           // this thread holds a block of tile t0 + u
#pragma unroll
    for (int u = 0; u < kHistTilesPerCta; ++u) {
      have[u] = false;
      if (t0 + u >= n_blocks) continue;                   // uniform over the CTA: the table's last CTA may hold one tile
      const MultiDesc d = descs[multi_find(descs, n_desc, t0 + u)];
      const size_t i = (t0 + u - d.first_cta) * kHistThreads + threadIdx.x;
      slot[u] = d.slot;
      have[u] = i < d.n_units;
      if (have[u]) blk[u].load(d.x, i);                    // both loads issued before either block is binned
    }
    __syncthreads();
    uint32_t mx[kHistTilesPerCta];
#pragma unroll
    for (int u = 0; u < kHistTilesPerCta; ++u) mx[u] = have[u] ? bin_block(blk[u], s_hist + u * nbins) : 0u;
#pragma unroll
    for (int u = 0; u < kHistTilesPerCta; ++u) {
      if (t0 + u >= n_blocks) break;
      const uint32_t m = block_max<kHistThreads>(mx[u]);
      if (threadIdx.x == 0 && m != 0u) atomicMax(max_slot + slot[u], m);
      __syncthreads();                                     // block_max's scratch is reused by the next tile; bins complete
      unsigned long long *row = hist + (size_t)slot[u] * (size_t)nbins;
      for (int b = threadIdx.x; b < nbins; b += kHistThreads) {
        const uint32_t c = s_hist[u * nbins + b];
        if (c) atomicAdd(&row[b], (unsigned long long)c);
      }
    }
    return;
  }
  __syncthreads();
  uint32_t mx = 0;
  for (size_t i = (size_t)blockIdx.x * kHistThreads + threadIdx.x; i < n_blocks; i += (size_t)gridDim.x * kHistThreads) {
    Block<Tag, VB> b;
    b.load(x, i);
    mx = max(mx, bin_block(b, s_hist));
  }
  mx = block_max<kHistThreads>(mx);
  if (threadIdx.x == 0 && mx != 0u) atomicMax(max_slot, mx);
  __syncthreads();
  for (int b = threadIdx.x; b < nbins; b += kHistThreads) {
    const uint32_t c = s_hist[b];
    if (c) atomicAdd(&hist[b], (unsigned long long)c);
  }
}

}  // namespace b200q

using namespace b200q;

extern "C" int b200q_nvfp4_block_log2_hist(const void *x, int dtype, size_t n_blocks, float log2_min,
                                           float log2_max, int nbins, long long *hist,
                                           float *running_max_slot, b200q_stream_t stream) {
  if (n_blocks == 0) return B200Q_OK;
  B200Q_REQUIRE(x != nullptr && hist != nullptr && running_max_slot != nullptr, "null pointer");
  B200Q_REQUIRE(nbins > 0 && nbins <= 16384 && log2_max > log2_min, "bad histogram arguments");
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x);
  B200Q_REQUIRE(ax % 16 == 0, "x must be 16-byte aligned");
  size_t grid = (n_blocks + kHistThreads - 1) / kHistThreads;
  const size_t cap = (size_t)sm_count() * 4;
  if (grid > cap) grid = cap;
  const size_t smem = (size_t)nbins * sizeof(uint32_t);
  const float range = log2_max - log2_min;
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  unsigned long long *h = reinterpret_cast<unsigned long long *>(hist);
  uint32_t *ms = reinterpret_cast<uint32_t *>(running_max_slot);
#define LAUNCH(VB_)                                                                                \
  do {                                                                                             \
    auto kern = block_log2_hist_kernel<Tag, VB_>;                                                  \
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    kern<<<(unsigned)grid, kHistThreads, smem, st>>>(xb, n_blocks, nullptr, 0, log2_min, range, nbins, h, ms); \
  } while (0)
  B200Q_DISPATCH_DTYPE(dtype, Tag, if (ax % 32 == 0) LAUNCH(32); else LAUNCH(16));
#undef LAUNCH
  return check_launch("block_log2_hist_kernel");
}

extern "C" int b200q_nvfp4_block_log2_hist_multi(const void *descs, int n_desc, size_t total_ctas, int dtype,
                                                 float log2_min, float log2_max, int nbins, long long *hist,
                                                 float *running_max, b200q_stream_t stream) {
  if (n_desc == 0 || total_ctas == 0) return B200Q_OK;
  B200Q_REQUIRE(descs != nullptr && hist != nullptr && running_max != nullptr && n_desc > 0, "null pointer");
  B200Q_REQUIRE(nbins > 0 && nbins <= 16384 && log2_max > log2_min, "bad histogram arguments");
  B200Q_REQUIRE(total_ctas <= 0x7fffffffu, "too many CTAs");
  const size_t smem = (size_t)kHistTilesPerCta * nbins * sizeof(uint32_t);   // one histogram per tile of a CTA
  const size_t grid = (total_ctas + kHistTilesPerCta - 1) / kHistTilesPerCta;
  const float range = log2_max - log2_min;
  const MultiDesc *dd = static_cast<const MultiDesc *>(descs);
  unsigned long long *h = reinterpret_cast<unsigned long long *>(hist);
  uint32_t *ms = reinterpret_cast<uint32_t *>(running_max);
  cudaStream_t st = (cudaStream_t)stream;
  B200Q_DISPATCH_DTYPE(dtype, Tag, {
    auto kern = block_log2_hist_kernel<Tag, 32>;          // table entries are 32-byte aligned (ops.TensorTable)
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<(unsigned)grid, kHistThreads, smem, st>>>(nullptr, total_ctas, dd, n_desc, log2_min, range, nbins, h, ms);
  });
  return check_launch("block_log2_hist_kernel<grouped>");
}

extern "C" int b200q_histogram(const void *x, int dtype, size_t n, int take_abs,
                               const float *range_max, int nbins, float *hist,
                               b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n == 0, "x is null");
  B200Q_REQUIRE(range_max != nullptr && hist != nullptr && nbins > 0 && nbins < (1 << 23), "bad histogram arguments");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_histogram<Tag>(x, n, take_abs, range_max, nbins, nullptr, hist, nullptr, (cudaStream_t)stream));
  return B200Q_OK;
}

extern "C" int b200q_histogram_ex(const void *x, int dtype, size_t n, int take_abs, const float *range_max, int nbins,
                                  const void *plan_state, float *hist, uint32_t *pattern_scratch,
                                  b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n == 0, "x is null");
  B200Q_REQUIRE(hist != nullptr && (plan_state != nullptr || (range_max != nullptr && nbins > 0 && nbins < (1 << 23))),
                "bad histogram arguments");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_histogram<Tag>(x, n, take_abs, range_max, nbins,
                                                    static_cast<const HistPlan *>(plan_state), hist, pattern_scratch,
                                                    (cudaStream_t)stream));
  return B200Q_OK;
}

extern "C" int b200q_hist_plan(const float *batch_amax, int nbins0, int capacity, void *plan_state,
                               b200q_stream_t stream) {
  B200Q_REQUIRE(batch_amax != nullptr && plan_state != nullptr, "null pointer");
  B200Q_REQUIRE(nbins0 > 0 && capacity >= nbins0 && capacity < (1 << 23), "bad histogram plan arguments");
  static_assert(sizeof(HistPlan) == 32, "HistPlan is 8 x 4 bytes (b200quant.h)");
  hist_plan_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(batch_amax, nbins0, capacity, static_cast<HistPlan *>(plan_state));
  return check_launch("hist_plan_kernel");
}

extern "C" int b200q_histogram_planned(const void *x, int dtype, size_t n, int take_abs, const void *plan_state,
                                       float *hist, b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n == 0, "x is null");
  B200Q_REQUIRE(plan_state != nullptr && hist != nullptr, "null pointer");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_histogram<Tag>(x, n, take_abs, nullptr, 0, static_cast<const HistPlan *>(plan_state),
                                                    hist, nullptr, (cudaStream_t)stream));
  return B200Q_OK;
}
