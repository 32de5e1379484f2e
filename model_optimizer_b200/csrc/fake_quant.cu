// fake_quant.cu -- fused fake-quant forward (scale -> round -> clamp -> dequant in ONE pass) for
// integer and FP8-E4M3 formats, per-tensor and per-channel.  4 B of HBM traffic per bf16
// element (2 read + 2 write); everything else lives in registers.
//
// Reference semantics (bit-exact):
//   integer : kernels/quantization/gemm/tensor_quant_gpu.cu:43-140  (fake_tensor_quant_device)
//   fp8     : kernels/quantization/gemm/tensor_quant_gpu_fp8.cu:36-107 (fake_e4m3fy[_with_axis])
#include "intq.cuh"

namespace b200q {

constexpr int kEwThreads = 256;

// x / d for 0 <= x < 2^31 with a precomputed multiplier (host side), 2 instructions on device
struct FastDivMod {
  uint32_t d, mul, shr;
  FastDivMod() : d(1), mul(0), shr(0) {}
  explicit FastDivMod(uint32_t d_) : d(d_), mul(0), shr(0) {
    if (d_ > 1) {
      uint32_t lg = 0;
      while ((1ull << lg) < d_) ++lg;  // ceil(log2 d)
      const uint32_t p = 31 + lg;
      mul = (uint32_t)(((1ull << p) + d_ - 1) / d_);
      shr = p - 32;
    }
  }
  __device__ __forceinline__ uint32_t div(uint32_t x) const {
    return d == 1 ? x : (__umulhi(x, mul) >> shr);
  }
  __device__ __forceinline__ uint32_t mod(uint32_t x) const { return x - div(x) * d; }
};

// how a vector finds its amax
enum : int { kPerTensor = 0, kPerRowVec = 1, kPerElem = 2, kPerRowTile = 3 };

struct ChannelMap {
  int mode;
  FastDivMod vecs_per_row;  // kPerRowVec: row = vec_idx / vecs_per_row; kPerRowTile: row = tile / tiles_per_row
  FastDivMod n_amax_div;    //             channel = row % n_amax
  size_t outer, n_amax;     // kPerElem : channel = (elem / outer) % n_amax
};

// ---------------------------------------------------------------------------------------------
// integer op
// ---------------------------------------------------------------------------------------------
struct IntParams {
  const void *amax;
  int amax_dtype;
  float max_bound, min_bound;
};

// plain torch-style cast round trip (amax == None): overflow -> NaN
__device__ __forceinline__ float fp8_torch_roundtrip(float v) {
  return e4m3_bits_to_f32(f32_to_e4m3fn_torch(v));
}

// ---------------------------------------------------------------------------------------------
// generic elementwise kernel.  KIND 0: integer, KIND 1: fp8 (scaled), KIND 2: fp8 torch cast
// ---------------------------------------------------------------------------------------------
template <typename Tag, int VB, int UNROLL, int KIND, int MODE>
__global__ void __launch_bounds__(kEwThreads)
    fake_quant_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t nvec,
                      size_t num_tiles, IntParams ip, ChannelMap cm) {
  constexpr int EPV = VB / Elem<Tag>::SIZE;
  const Vec<VB> *xv = reinterpret_cast<const Vec<VB> *>(x);
  Vec<VB> *yv = reinterpret_cast<Vec<VB> *>(y);

  pdl_launch_dependents();
  pdl_wait();
  IntQ is;
  Fp8Scale fs;
  if constexpr (MODE == kPerTensor && KIND != 2) {
    const float amax = load_scalar(ip.amax, ip.amax_dtype, 0);
    if constexpr (KIND == 0) is.setup(amax, ip.max_bound, ip.min_bound);
    else fs.setup(amax, ip.max_bound != 0.f);
  }

  for (size_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const size_t base = tile * (size_t)(kEwThreads * UNROLL) + threadIdx.x;
    if constexpr (MODE == kPerRowTile && KIND != 2) {  // the whole tile lies in one row: one setup per CTA tile
      const uint32_t row = cm.vecs_per_row.div((uint32_t)tile);
      const float amax = load_scalar(ip.amax, ip.amax_dtype, cm.n_amax_div.mod(row));
      if constexpr (KIND == 0) is.setup(amax, ip.max_bound, ip.min_bound);
      else fs.setup(amax, ip.max_bound != 0.f);
    }
    Vec<VB> v[UNROLL];
    float row_amax[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = base + (size_t)u * kEwThreads;
      row_amax[u] = 0.f;
      if (i < nvec) {
        v[u] = ldg_stream(xv + i);
        if constexpr (MODE == kPerRowVec && KIND != 2) {  // amax fetched with the data, not after it
          const uint32_t row = cm.vecs_per_row.div((uint32_t)i);
          row_amax[u] = load_scalar(ip.amax, ip.amax_dtype, cm.n_amax_div.mod(row));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = base + (size_t)u * kEwThreads;
      if (i >= nvec) continue;
      float f[EPV];
      vec_to_floats<Tag, VB>(v[u], f);
      if constexpr (MODE == kPerRowVec && KIND != 2) {
        if constexpr (KIND == 0) is.setup(row_amax[u], ip.max_bound, ip.min_bound);
        else fs.setup(row_amax[u], ip.max_bound != 0.f);
      }
      if constexpr (MODE == kPerElem && KIND != 2) {
#pragma unroll
        for (int e = 0; e < EPV; e += 2) {
          const size_t e0 = i * EPV + e;
          const float a0 = load_scalar(ip.amax, ip.amax_dtype, (e0 / cm.outer) % cm.n_amax);
          const float a1 = load_scalar(ip.amax, ip.amax_dtype, ((e0 + 1) / cm.outer) % cm.n_amax);
          if constexpr (KIND == 0) {
            is.setup(a0, ip.max_bound, ip.min_bound);
            f[e] = is.apply_ref(f[e]);
            is.setup(a1, ip.max_bound, ip.min_bound);
            f[e + 1] = is.apply_ref(f[e + 1]);
          } else {
            Fp8Scale s0, s1;
            s0.setup(a0, ip.max_bound != 0.f);
            s1.setup(a1, ip.max_bound != 0.f);
            s0.apply2(f[e], f[e + 1], s1);
          }
        }
      } else if constexpr (KIND == 0) {
        is.template apply_vec<EPV>(f);
      } else if constexpr (KIND == 1) {
#pragma unroll
        for (int e = 0; e < EPV; e += 2) fs.apply2(f[e], f[e + 1]);
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) f[e] = fp8_torch_roundtrip(f[e]);
      }
      Vec<VB> o;
      floats_to_vec<Tag, VB>(f, o);
      stg(yv + i, o);
    }
  }
}

// scalar kernel for ragged ends / unaligned tensors: element range [begin, end)
template <typename Tag, int KIND>
__global__ void __launch_bounds__(kEwThreads)
    fake_quant_scalar_kernel(const void *__restrict__ x, void *__restrict__ y, size_t begin,
                             size_t end, IntParams ip, size_t outer, size_t n_amax) {
  for (size_t i = begin + blockIdx.x * (size_t)kEwThreads + threadIdx.x; i < end;
       i += (size_t)gridDim.x * kEwThreads) {
    float v = Elem<Tag>::load1(x, i);
    if constexpr (KIND == 2) {
      v = fp8_torch_roundtrip(v);
    } else {
      const float amax = load_scalar(ip.amax, ip.amax_dtype, n_amax == 1 ? 0 : (i / outer) % n_amax);
      if constexpr (KIND == 0) {
        IntQ is;
        is.setup(amax, ip.max_bound, ip.min_bound);
        v = is.apply_ref(v);
      } else {
        Fp8Scale fs;
        fs.setup(amax, ip.max_bound != 0.f);
        float dummy = 0.f;
        fs.apply2(v, dummy);
      }
    }
    Elem<Tag>::store1(y, i, v);
  }
}

template <typename Tag, int KIND>
static int launch_fake_quant(const void *x, void *y, size_t n, IntParams ip, size_t n_amax,
                             size_t outer, cudaStream_t st) {
  if (n == 0) return B200Q_OK;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), ay = reinterpret_cast<uintptr_t>(y);
  B200Q_REQUIRE(ax % Elem<Tag>::SIZE == 0 && ay % Elem<Tag>::SIZE == 0, "tensor not element-aligned");
  int vb = tuning("vec_bytes", 32);
  int unroll = tuning("ew_unroll", 2);
  if (vb == 32 && (ax % 32 != 0 || ay % 32 != 0)) vb = 16;
  const bool aligned = (ax % vb == 0) && (ay % vb == 0);

  ChannelMap cm;
  cm.mode = kPerTensor;
  cm.outer = outer;
  cm.n_amax = n_amax;
  size_t nvec = 0;
  if (aligned) {
    const size_t epv = vb / Elem<Tag>::SIZE;
    nvec = n / epv;
    if (n_amax > 1 && KIND != 2) {
      if (outer % epv == 0 && nvec < 0x7fffffffull && outer / epv < 0x7fffffffull && n_amax < 0x7fffffffull) {
        const size_t vpr = outer / epv;
        cm.n_amax_div = FastDivMod((uint32_t)n_amax);
        if (vpr % ((size_t)kEwThreads * 2) == 0 && unroll == 2) {
          cm.mode = kPerRowTile;
          cm.vecs_per_row = FastDivMod((uint32_t)(vpr / (kEwThreads * 2)));
        } else if (vpr % (size_t)kEwThreads == 0) {
          cm.mode = kPerRowTile;
          unroll = 1;
          cm.vecs_per_row = FastDivMod((uint32_t)(vpr / kEwThreads));
        } else {
          cm.mode = kPerRowVec;
          cm.vecs_per_row = FastDivMod((uint32_t)vpr);
        }
      } else {
        cm.mode = kPerElem;
      }
    }
  }
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  uint8_t *yb = static_cast<uint8_t *>(y);
  if (nvec > 0) {
    const size_t tiles = (nvec + (size_t)kEwThreads * unroll - 1) / ((size_t)kEwThreads * unroll);
    B200Q_REQUIRE(tiles <= 0x7fffffffu, "tensor too large");
    const unsigned grid = (unsigned)tiles;
#define LAUNCH(VB_, U_, MODE_)                                                                     \
  launch_pdl(fake_quant_kernel<Tag, VB_, U_, KIND, MODE_>, dim3(grid), dim3(kEwThreads), 0, st, xb, yb, nvec, tiles, ip, cm)
#define LAUNCH_MODE(VB_, U_)                                                                       \
  do {                                                                                             \
    if (cm.mode == kPerTensor) LAUNCH(VB_, U_, kPerTensor);                                        \
    else if (cm.mode == kPerRowVec) LAUNCH(VB_, U_, kPerRowVec);                                   \
    else if (cm.mode == kPerRowTile) LAUNCH(VB_, U_, kPerRowTile);                                 \
    else LAUNCH(VB_, U_, kPerElem);                                                                \
  } while (0)
    if (vb == 32) {
      if (unroll == 1) LAUNCH_MODE(32, 1);
      else if (unroll == 4) LAUNCH_MODE(32, 4);
      else LAUNCH_MODE(32, 2);
    } else {
      if (unroll == 1) LAUNCH_MODE(16, 1);
      else if (unroll == 4) LAUNCH_MODE(16, 4);
      else LAUNCH_MODE(16, 2);
    }
#undef LAUNCH_MODE
#undef LAUNCH
    int rc = check_launch("fake_quant_kernel");
    if (rc != B200Q_OK) return rc;
  }
  const size_t done = nvec * (vb / Elem<Tag>::SIZE);
  if (done < n) {
    const size_t rem = n - done;
    size_t grid = (rem + kEwThreads - 1) / kEwThreads;
    const size_t cap = (size_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    fake_quant_scalar_kernel<Tag, KIND><<<(unsigned)grid, kEwThreads, 0, st>>>(x, y, done, n, ip, outer, n_amax);
    return check_launch("fake_quant_scalar_kernel");
  }
  return B200Q_OK;
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_fake_quant_int(const void *x, void *y, int dtype, size_t n, const void *amax,
                         int amax_dtype, size_t n_amax, size_t outer, int num_bits,
                         int is_unsigned, int narrow_range, b200q_stream_t stream) {
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n == 0, "null tensor");
  B200Q_REQUIRE(amax != nullptr && dtype_ok(amax_dtype), "amax is null or has a bad dtype");
  B200Q_REQUIRE(n_amax >= 1 && outer >= 1, "n_amax and outer must be >= 1");
  B200Q_REQUIRE(num_bits >= 1 && num_bits + (is_unsigned ? 1 : 0) <= 24, "unsupported num_bits %d", num_bits);
  IntParams ip;
  ip.amax = amax;
  ip.amax_dtype = amax_dtype;
  // bits_to_bound (tensor_quant_gpu.cu:38-41) and the bound arithmetic of the kernel (:69-71)
  const float bound = (float)((1 << (num_bits - 1 + (is_unsigned ? 1 : 0))) - 1);
  ip.max_bound = bound;
  ip.min_bound = -(bound + (narrow_range ? 0.f : 1.f));
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return (launch_fake_quant<Tag, 0>(x, y, n, ip, n_amax, outer, (cudaStream_t)stream)));
  return B200Q_OK;
}

static int fake_quant_fp8_impl(const void *x, void *y, int dtype, size_t n, const void *amax, int amax_dtype,
                               size_t n_amax, size_t outer, bool eager, b200q_stream_t stream) {
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n == 0, "null tensor");
  IntParams ip;
  ip.amax = amax;
  ip.amax_dtype = amax_dtype;
  ip.max_bound = eager ? 1.0f : 0.f;  // the FP8 kernels read max_bound as the "eager scale rule" flag
  ip.min_bound = 0.f;
  if (amax == nullptr) {
    B200Q_DISPATCH_DTYPE(dtype, Tag,
                         return (launch_fake_quant<Tag, 2>(x, y, n, ip, 1, 1, (cudaStream_t)stream)));
    return B200Q_OK;
  }
  B200Q_REQUIRE(dtype_ok(amax_dtype), "bad amax dtype");
  B200Q_REQUIRE(n_amax >= 1 && outer >= 1, "n_amax and outer must be >= 1");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return (launch_fake_quant<Tag, 1>(x, y, n, ip, n_amax, outer, (cudaStream_t)stream)));
  return B200Q_OK;
}

int b200q_fake_quant_fp8(const void *x, void *y, int dtype, size_t n, const void *amax,
                         int amax_dtype, size_t n_amax, size_t outer, b200q_stream_t stream) {
  return fake_quant_fp8_impl(x, y, dtype, n, amax, amax_dtype, n_amax, outer, false, stream);
}

int b200q_fake_quant_fp8_eager(const void *x, void *y, int dtype, size_t n, const void *amax,
                               int amax_dtype, size_t n_amax, size_t outer, b200q_stream_t stream) {
  return fake_quant_fp8_impl(x, y, dtype, n, amax, amax_dtype, n_amax, outer, true, stream);
}

}  // extern "C"
