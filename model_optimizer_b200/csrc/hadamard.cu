// hadamard.cu -- normalized fast Walsh-Hadamard transform over contiguous blocks of B = 2^k elements (k = 0..15), and
// the fused rotate -> NVFP4 fake quant (-> rotate back) pass of a rotated NVFP4 quantizer.
//
// Arithmetic (restated by tools/hadamard_oracle.py): load and widen to fp32; stages s = 0 .. k-1 in ascending order,
// stage s pairs element i with i | 2^s (bit s of i clear) and maps (a, b) -> (a + b, a - b), every add a separate
// fp32 round-to-nearest (__fadd_rn / __fsub_rn: nothing is contracted); one multiply by scale = fl32(B^-0.5) after the
// last stage; one RNE rounding to the output type.  Every path below runs the stages in that order on the same values,
// so all of them give the same bits.
//
// Layout: one thread owns one group of 16 consecutive elements (one 32-byte vector for 16-bit types, two for fp32).
// Stages 0-3 run in its registers, stages 4-8 through __shfl_xor_sync (a warp spans 512 elements), and for B > 512 the
// CTA owns one whole block and the stages from 9 up exchange through shared memory in fp32 (B * 4 bytes: 128 KB at
// B = 32768), in passes of up to 3 stages over groups of 8 values.  B < 16: a thread holds 16 / B blocks.
// Pointers that are not 32-byte aligned, or an element count that is not a multiple of 16, take the scalar load /
// store path of the same kernel (the arithmetic is unchanged).
//
// The rotated NVFP4 pass rounds the transform to T, runs the NVFP4 dynamic block-16 fake quant of nvfp4.cu on those
// 16 values (qdq_block / DynScale, block16.cuh: the 16-element group IS the NVFP4 block) and, for rotate_back,
// transforms the result again: bit-identical to hadamard -> fake_quant_nvfp4 -> hadamard, moving each element through
// HBM once instead of three times.
#include <math.h>

#include <algorithm>

#include "block16.cuh"

namespace b200q {

constexpr int kHadRegLog = 4;        // stages in registers (16 elements per thread)
constexpr int kHadWarpLog = 9;       // stages within a warp (32 x 16 elements)
constexpr int kHadMaxLog = 15;       // B <= 32768
constexpr int kHadPassLog = 3;       // stages per shared-memory pass (8 values per thread and group)
constexpr int kHadThreads = 256;     // CTA size for B <= 512
constexpr int kHadMaxThreads = 512;  // CTA size cap for B > 512 (a thread then holds up to 4 groups)

// stages 0 .. min(k, 4) - 1 on the 16 values of one group
__device__ __forceinline__ void had_reg_stages(float (&f)[kBlk], int k) {
#pragma unroll
  for (int s = 0; s < kHadRegLog; ++s) {
    if (s < k) {
#pragma unroll
      for (int i = 0; i < kBlk; ++i) {
        if (!(i & (1 << s))) {
          const float a = f[i], b = f[i | (1 << s)];
          f[i] = __fadd_rn(a, b);
          f[i | (1 << s)] = __fsub_rn(a, b);
        }
      }
    }
  }
}

// stages 4 .. min(k, 9) - 1: bit s of the element index is bit s - 4 of the lane (groups are lane-consecutive)
__device__ __forceinline__ void had_warp_stages(float (&f)[kBlk], int k) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int s = kHadRegLog; s < kHadWarpLog; ++s) {
    if (s < k) {
      const int m = 1 << (s - kHadRegLog);
      const bool upper = (lane & m) != 0;
#pragma unroll
      for (int i = 0; i < kBlk; ++i) {
        const float p = __shfl_xor_sync(0xffffffffu, f[i], m);
        f[i] = upper ? __fsub_rn(p, f[i]) : __fadd_rn(f[i], p);
      }
    }
  }
}

// stages b0 .. b0 + NB - 1 over the n (a multiple of 2^(b0 + NB)) fp32 values in shared memory: each thread takes
// groups of 2^NB values closed under those index bits
template <int NB> __device__ __forceinline__ void had_smem_pass(float *s, int b0, unsigned n) {
  const unsigned lo_mask = (1u << b0) - 1u;
  for (unsigned g = threadIdx.x; g < (n >> NB); g += blockDim.x) {
    const unsigned base = (g & lo_mask) | ((g & ~lo_mask) << NB);
    float v[1 << NB];
#pragma unroll
    for (int j = 0; j < (1 << NB); ++j) v[j] = s[base + ((unsigned)j << b0)];
#pragma unroll
    for (int t = 0; t < NB; ++t) {
#pragma unroll
      for (int j = 0; j < (1 << NB); ++j) {
        if (!(j & (1 << t))) {
          const float a = v[j], b = v[j | (1 << t)];
          v[j] = __fadd_rn(a, b);
          v[j | (1 << t)] = __fsub_rn(a, b);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < (1 << NB); ++j) s[base + ((unsigned)j << b0)] = v[j];
  }
}

// stages 9 .. k-1 through shared memory: the CTA holds exactly one block, group v of thread t is group
// v * blockDim.x + t of the block, and s has room for its 2^k fp32 values
template <int VPT> __device__ __forceinline__ void had_smem_stages(float (&f)[VPT][kBlk], float *s, int k) {
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    float4 *p = reinterpret_cast<float4 *>(s + ((size_t)v * blockDim.x + threadIdx.x) * kBlk);
#pragma unroll
    for (int i = 0; i < kBlk / 4; ++i) p[i] = make_float4(f[v][4 * i], f[v][4 * i + 1], f[v][4 * i + 2], f[v][4 * i + 3]);
  }
  const unsigned n = 1u << k;
  for (int b0 = kHadWarpLog; b0 < k; b0 += kHadPassLog) {
    __syncthreads();
    switch (min(kHadPassLog, k - b0)) {
    case 1: had_smem_pass<1>(s, b0, n); break;
    case 2: had_smem_pass<2>(s, b0, n); break;
    default: had_smem_pass<3>(s, b0, n); break;
    }
  }
  __syncthreads();
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    const float4 *p = reinterpret_cast<const float4 *>(s + ((size_t)v * blockDim.x + threadIdx.x) * kBlk);
#pragma unroll
    for (int i = 0; i < kBlk / 4; ++i) {
      const float4 q = p[i];
      f[v][4 * i] = q.x;
      f[v][4 * i + 1] = q.y;
      f[v][4 * i + 2] = q.z;
      f[v][4 * i + 3] = q.w;
    }
  }
  // the next writes to s are this thread's own slots, which no other thread reads after the barrier above
}

// the whole transform (without the scale) of the VPT groups a thread holds; SMEM for k > 9
template <int VPT, bool SMEM>
__device__ __forceinline__ void had_transform(float (&f)[VPT][kBlk], float *s, int k) {
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    had_reg_stages(f[v], k);
    had_warp_stages(f[v], k);
  }
  if constexpr (SMEM) had_smem_stages<VPT>(f, s, k);
}

// transform + scale + RNE rounding to T of the values in f, into b
template <typename Tag, int VPT, bool SMEM>
__device__ __forceinline__ void had_rotate(float (&f)[VPT][kBlk], Block<Tag, 32> (&b)[VPT], float *s, int k,
                                           float scale) {
  had_transform<VPT, SMEM>(f, s, k);
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
#pragma unroll
    for (int i = 0; i < kBlk; ++i) f[v][i] = __fmul_rn(f[v][i], scale);
    b[v].from_floats(f[v]);
  }
}

// MODE 0: y = H x (amax_slot: also folds max|y| of the rounded outputs into *amax_slot, the rule of
// amax_tensor_kernel); MODE 1: y = fake_quant_nvfp4(H x); MODE 2: y = H fake_quant_nvfp4(H x).
// vec: x and y are 32-byte aligned and n % 16 == 0 (vector loads / stores); otherwise element-wise, zero-filled past n.
template <typename Tag, int VPT, int MODE, bool SMEM>
__global__ void __launch_bounds__(SMEM ? kHadMaxThreads : kHadThreads)
    hadamard_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t n, int k, float scale, bool vec,
                    uint32_t *__restrict__ amax_slot, const void *__restrict__ gamax, int gamax_dtype) {
  extern __shared__ __align__(16) float s_had[];
  pdl_launch_dependents();
  pdl_wait();
  Block<Tag, 32> b[VPT];
  float f[VPT][kBlk];
  size_t q[VPT];
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    q[v] = ((size_t)blockIdx.x * VPT + v) * blockDim.x + threadIdx.x;
    if (vec) {
      if (q[v] * kBlk < n) {
        b[v].load(x, q[v]);
        b[v].to_floats(f[v]);
      } else {
#pragma unroll
        for (int i = 0; i < kBlk; ++i) f[v][i] = 0.0f;
      }
    } else {
#pragma unroll
      for (int i = 0; i < kBlk; ++i) {
        const size_t e = q[v] * kBlk + i;
        f[v][i] = e < n ? Elem<Tag>::load1(x, e) : 0.0f;
      }
    }
  }
  had_rotate<Tag, VPT, SMEM>(f, b, s_had, k, scale);
  if constexpr (MODE != 0) {
    DynScale ds;
    ds.setup(load_scalar(gamax, gamax_dtype, 0));
    const ExactDiv d6(ds.six_gs);
#pragma unroll
    for (int v = 0; v < VPT; ++v) {
      const uint32_t mb = b[v].prep_and_absmax_bits();
      qdq_block<Tag, 32>(b[v], ds.block_scale(dyn_block_max(b[v], mb), d6), mb < 0x7f800000u);
    }
    if constexpr (MODE == 2) {
#pragma unroll
      for (int v = 0; v < VPT; ++v) b[v].to_floats(f[v]);
      had_rotate<Tag, VPT, SMEM>(f, b, s_had, k, scale);
    }
  }
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    if (vec) {
      if (q[v] * kBlk < n) b[v].store(y, q[v]);
    } else {
#pragma unroll
      for (int i = 0; i < kBlk; ++i) {
        const size_t e = q[v] * kBlk + i;
        if (e >= n) continue;
        if constexpr (Elem<Tag>::SIZE == 2)
          reinterpret_cast<uint16_t *>(y)[e] = (uint16_t)(b[v].word(i / 2) >> (16 * (i & 1)));
        else
          reinterpret_cast<uint32_t *>(y)[e] = b[v].word(i);
      }
    }
  }
  if constexpr (MODE == 0) {
    if (amax_slot == nullptr) return;
    // groups past n hold zeros, which do not move the max
    uint32_t acc = 0;
#pragma unroll
    for (int v = 0; v < VPT; ++v)
#pragma unroll
      for (int w = 0; w < Block<Tag, 32>::WORDS; ++w) acc = absmax_acc<Tag>(acc, b[v].word(w));
    __shared__ uint32_t s_part[kHadMaxThreads / 32];
    uint32_t m = __reduce_max_sync(0xffffffffu, absmax_collapse<Tag>(acc));
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
      m = __reduce_max_sync(0xffffffffu, threadIdx.x < (blockDim.x >> 5) ? s_part[threadIdx.x] : 0u);
      if (threadIdx.x == 0 && m != 0u) {
        const uint32_t fb = Elem<Tag>::absbits_to_f32bits(m);
        if (fb > __ldcg(amax_slot)) atomicMax(amax_slot, fb);
      }
    }
  }
}

template <typename Tag, int VPT, int MODE, bool SMEM>
static int launch_hadamard_vpt(const void *x, void *y, size_t n, int k, bool vec, float *amax_slot, const void *gamax,
                               int gamax_dtype, unsigned threads, size_t grid, cudaStream_t st) {
  auto kern = hadamard_kernel<Tag, VPT, MODE, SMEM>;
  const size_t smem = SMEM ? (sizeof(float) << k) : 0;
  // the opt-in above 48 KB is a property of the function on the CURRENT device: set it on every such launch (a
  // host-side attribute write, no device work), so that a process running the op on several devices is covered
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("hadamard_kernel (shared-memory opt-in)");
  const float scale = (float)pow((double)(1u << k), -0.5);  // fl32(B ** -0.5)
  launch_pdl(kern, dim3((unsigned)grid), dim3(threads), smem, st, static_cast<const uint8_t *>(x),
             static_cast<uint8_t *>(y), n, k, scale, vec, reinterpret_cast<uint32_t *>(amax_slot), gamax, gamax_dtype);
  return check_launch("hadamard_kernel");
}

template <typename Tag, int MODE>
static int launch_hadamard(const void *x, void *y, size_t n, int k, float *amax_slot, const void *gamax,
                           int gamax_dtype, cudaStream_t st) {
  if (n == 0) return B200Q_OK;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), ay = reinterpret_cast<uintptr_t>(y);
  B200Q_REQUIRE(ax % Elem<Tag>::SIZE == 0 && ay % Elem<Tag>::SIZE == 0, "tensor not element-aligned");
  const bool vec = ax % 32 == 0 && ay % 32 == 0 && n % kBlk == 0;
  if (k <= kHadWarpLog) {
    const size_t grid = ((n + kBlk - 1) / kBlk + kHadThreads - 1) / kHadThreads;
    B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
    return launch_hadamard_vpt<Tag, 1, MODE, false>(x, y, n, k, vec, amax_slot, gamax, gamax_dtype, kHadThreads, grid,
                                                    st);
  }
  // one CTA per block of B: min(B / 16, 512) threads holding B / 16 / threads groups each
  const size_t groups = (size_t)1 << (k - 4);
  const unsigned threads = (unsigned)std::min(groups, (size_t)kHadMaxThreads);
  const size_t grid = n >> k;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  switch (groups / threads) {
  case 1: return launch_hadamard_vpt<Tag, 1, MODE, true>(x, y, n, k, vec, amax_slot, gamax, gamax_dtype, threads, grid, st);
  case 2: return launch_hadamard_vpt<Tag, 2, MODE, true>(x, y, n, k, vec, amax_slot, gamax, gamax_dtype, threads, grid, st);
  default: return launch_hadamard_vpt<Tag, 4, MODE, true>(x, y, n, k, vec, amax_slot, gamax, gamax_dtype, threads, grid, st);
  }
}

static int block_log2(size_t block_size) {
  for (int k = 0; k <= kHadMaxLog; ++k)
    if (block_size == ((size_t)1 << k)) return k;
  return -1;
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_hadamard(const void *x, void *y, int dtype, size_t n_rows, size_t row_len, size_t block_size,
                   float *amax_slot, b200q_stream_t stream) {
  const size_t n = n_rows * row_len;
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n == 0, "null tensor");
  B200Q_REQUIRE(x != y || n == 0, "the output must not alias the input");
  const int k = block_log2(block_size);
  B200Q_REQUIRE(k >= 0, "block_size must be a power of 2 no larger than 32768, got %zu", block_size);
  B200Q_REQUIRE(row_len % block_size == 0, "row_len %zu is not a multiple of block_size %zu", row_len, block_size);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_hadamard<Tag, 0>(x, y, n, k, amax_slot, nullptr, 0, (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_fake_quant_nvfp4_rotated(const void *x, void *y, int dtype, size_t n_rows, size_t row_len,
                                   size_t block_size, int rotate_back, const void *global_amax, int amax_dtype,
                                   b200q_stream_t stream) {
  const size_t n = n_rows * row_len;
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n == 0, "null tensor");
  B200Q_REQUIRE(x != y || n == 0, "the output must not alias the input");
  B200Q_REQUIRE(global_amax != nullptr && dtype_ok(amax_dtype), "global_amax is null or has a bad dtype");
  const int k = block_log2(block_size);
  B200Q_REQUIRE(k >= 0, "block_size must be a power of 2 no larger than 32768, got %zu", block_size);
  B200Q_REQUIRE(row_len % block_size == 0, "row_len %zu is not a multiple of block_size %zu", row_len, block_size);
  B200Q_REQUIRE(row_len % kBlk == 0, "row_len %zu is not a multiple of the NVFP4 block (16)", row_len);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return rotate_back ? launch_hadamard<Tag, 2>(x, y, n, k, nullptr, global_amax, amax_dtype,
                                                                    (cudaStream_t)stream)
                                          : launch_hadamard<Tag, 1>(x, y, n, k, nullptr, global_amax, amax_dtype,
                                                                    (cudaStream_t)stream));
  return B200Q_OK;
}

}  // extern "C"
