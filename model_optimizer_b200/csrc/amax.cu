// amax.cu -- calibration collect: per-tensor / per-row(block) / per-column |x| maxima, column
// abs-sums and amax export.  All HBM-bound: 2 B (bf16) read per element, outputs negligible.
//
// Reference semantics: reduce_amax = max(|max(x)|, |min(x)|) == max|x| with NaN propagation
// (quantization/utils/core_utils.py:147-183); MaxCalibrator keeps the running elementwise max of
// it across batches (quantization/calib/max.py:53-86).  Here both happen in one pass: the kernel
// folds its result into the fp32 "amax slot" with an unsigned atomic max on the bit pattern.
#include <type_traits>

#include "common.cuh"

namespace b200q {

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------
// per-tensor
// ---------------------------------------------------------------------------------------------
template <typename Tag, int VB, int UNROLL>
__global__ void __launch_bounds__(kThreads)
    amax_tensor_kernel(const uint8_t *__restrict__ x, size_t head, size_t nvec, size_t tail,
                       size_t num_tiles, uint32_t *__restrict__ slot) {
  constexpr int EPV = VB / Elem<Tag>::SIZE;
  const Vec<VB> *xv = reinterpret_cast<const Vec<VB> *>(x + head * Elem<Tag>::SIZE);
  uint32_t acc = 0;
  pdl_launch_dependents();
  pdl_wait();

  for (size_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const size_t base = tile * (size_t)(kThreads * UNROLL) + threadIdx.x;
    Vec<VB> v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = base + (size_t)u * kThreads;
      if (i < nvec) {
        v[u] = ldg_stream(xv + i);
      } else {
#pragma unroll
        for (int w = 0; w < Vec<VB>::WORDS; ++w) v[u].r[w] = 0u;
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
#pragma unroll
      for (int w = 0; w < Vec<VB>::WORDS; ++w) acc = absmax_acc<Tag>(acc, v[u].r[w]);
  }
  uint32_t m = absmax_collapse<Tag>(acc);

  // ragged ends (unaligned base pointer / n not a multiple of the vector): last CTA, scalar
  if (blockIdx.x == gridDim.x - 1) {
    const uint32_t one_mask = Elem<Tag>::SIZE == 2 ? 0x7fffu : 0x7fffffffu;
    for (size_t i = threadIdx.x; i < head + tail; i += kThreads) {
      const size_t e = i < head ? i : (head + nvec * EPV + (i - head));
      uint32_t b;
      if constexpr (Elem<Tag>::SIZE == 2)
        b = reinterpret_cast<const uint16_t *>(x)[e];
      else
        b = reinterpret_cast<const uint32_t *>(x)[e];
      m = max(m, b & one_mask);
    }
  }

  m = block_max<kThreads>(m);
  if (threadIdx.x == 0 && m != 0u) atomicMax(slot, Elem<Tag>::absbits_to_f32bits(m));
}

// per-tensor over a table of tensors: CTA -> (tensor, 32 KB tile); one atomicMax per CTA into that tensor's slot
template <typename Tag, int VB, int UNROLL>
__global__ void __launch_bounds__(kThreads)
    amax_tensor_multi_kernel(const MultiDesc *__restrict__ descs, int n_desc, uint32_t *__restrict__ slots) {
  pdl_launch_dependents();
  pdl_wait();
  const MultiDesc d = descs[multi_find(descs, n_desc)];
  const Vec<VB> *xv = reinterpret_cast<const Vec<VB> *>(d.x);
  const size_t base = (size_t)(blockIdx.x - d.first_cta) * (size_t)(kThreads * UNROLL) + threadIdx.x;
  Vec<VB> v[UNROLL];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * kThreads;
    if (i < d.n_units) {
      v[u] = ldg_stream(xv + i);
    } else {
#pragma unroll
      for (int w = 0; w < Vec<VB>::WORDS; ++w) v[u].r[w] = 0u;
    }
  }
  uint32_t acc = 0;
#pragma unroll
  for (int u = 0; u < UNROLL; ++u)
#pragma unroll
    for (int w = 0; w < Vec<VB>::WORDS; ++w) acc = absmax_acc<Tag>(acc, v[u].r[w]);
  uint32_t m = block_max<kThreads>(absmax_collapse<Tag>(acc));
  if (threadIdx.x == 0 && m != 0u) atomicMax(slots + d.slot, Elem<Tag>::absbits_to_f32bits(m));
}

// ---------------------------------------------------------------------------------------------
// per-tensor, TMA variant: persistent CTAs stream 16-32 KB tiles through a shared-memory ring with
// cp.async.bulk (UBLKCP) + mbarrier transaction counts; one elected thread issues the copies, all
// threads reduce from shared memory.  Selected with the "amax_tma" tuning knob (see DESIGN.md 5 for
// its comparison with the vector-load kernel above).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "B200Q_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra B200Q_DONE;\n"
      "bra B200Q_WAIT;\n"
      "B200Q_DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

constexpr int kTmaMaxStages = 8;

template <typename Tag>
__global__ void __launch_bounds__(kThreads)
    amax_tensor_tma_kernel(const uint8_t *__restrict__ x, size_t head, size_t body_bytes, size_t tail,
                           size_t n_total, size_t num_tiles, uint32_t tile_bytes, int stages,
                           uint32_t *__restrict__ slot) {
  extern __shared__ __align__(128) uint8_t s_ring[];
  __shared__ __align__(8) uint64_t s_full[kTmaMaxStages];
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int k = 0; k < stages; ++k) mbar_init(&s_full[k], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const uint8_t *body = x + head * Elem<Tag>::SIZE;
  const size_t my_tiles = num_tiles > blockIdx.x ? (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  auto tile_size = [&](size_t k) -> uint32_t {
    const size_t off = (blockIdx.x + k * (size_t)gridDim.x) * (size_t)tile_bytes;
    const size_t rem = body_bytes - off;
    return (uint32_t)(rem < tile_bytes ? rem : tile_bytes);
  };
  auto issue = [&](size_t k) {
    const int st = (int)(k % stages);
    const uint32_t bytes = tile_size(k);
    mbar_expect_tx(&s_full[st], bytes);
    bulk_g2s(s_ring + (size_t)st * tile_bytes, body + (blockIdx.x + k * (size_t)gridDim.x) * (size_t)tile_bytes, bytes,
             &s_full[st]);
  };
  if (tid == 0)
    for (size_t k = 0; k < my_tiles && k < (size_t)stages; ++k) issue(k);

  uint32_t acc = 0;
  for (size_t k = 0; k < my_tiles; ++k) {
    const int st = (int)(k % stages);
    mbar_wait(&s_full[st], (uint32_t)((k / stages) & 1));
    const uint32_t nv = tile_size(k) / 16;
    const uint4 *sv = reinterpret_cast<const uint4 *>(s_ring + (size_t)st * tile_bytes);
    for (uint32_t v = tid; v < nv; v += kThreads) {
      const uint4 q = sv[v];
      acc = absmax_acc<Tag>(acc, q.x);
      acc = absmax_acc<Tag>(acc, q.y);
      acc = absmax_acc<Tag>(acc, q.z);
      acc = absmax_acc<Tag>(acc, q.w);
    }
    __syncthreads();  // every thread is done with this stage before it is refilled
    if (tid == 0 && k + stages < my_tiles) issue(k + stages);
  }
  uint32_t m = absmax_collapse<Tag>(acc);
  if (blockIdx.x == gridDim.x - 1) {  // ragged ends, scalar
    const uint32_t one_mask = Elem<Tag>::SIZE == 2 ? 0x7fffu : 0x7fffffffu;
    const size_t body_elems = body_bytes / Elem<Tag>::SIZE;
    for (size_t i = tid; i < head + tail; i += kThreads) {
      const size_t e = i < head ? i : (head + body_elems + (i - head));
      uint32_t b;
      if constexpr (Elem<Tag>::SIZE == 2) b = reinterpret_cast<const uint16_t *>(x)[e];
      else b = reinterpret_cast<const uint32_t *>(x)[e];
      m = max(m, b & one_mask);
    }
  }
  (void)n_total;
  m = block_max<kThreads>(m);
  if (tid == 0 && m != 0u) atomicMax(slot, Elem<Tag>::absbits_to_f32bits(m));
}

template <typename Tag>
static int launch_amax_tensor_tma(const void *x, size_t n, float *slot, cudaStream_t st) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
  size_t head = ((size_t)16 - addr % 16) % 16 / Elem<Tag>::SIZE;
  if (head > n) head = n;
  const size_t body_elems = (n - head) / (16 / Elem<Tag>::SIZE) * (16 / Elem<Tag>::SIZE);
  const size_t body_bytes = body_elems * Elem<Tag>::SIZE;
  const size_t tail = n - head - body_elems;
  const uint32_t tile_bytes = (uint32_t)tuning("tma_tile_kb", 16) * 1024u;
  int stages = tuning("tma_stages", 4);
  if (stages < 1) stages = 1;
  if (stages > kTmaMaxStages) stages = kTmaMaxStages;
  size_t tiles = (body_bytes + tile_bytes - 1) / tile_bytes;
  size_t grid = (size_t)sm_count() * tuning("tma_ctas_per_sm", 2);
  if (grid > tiles) grid = tiles;
  if (grid == 0) grid = 1;
  const size_t smem = (size_t)stages * tile_bytes;
  auto kern = amax_tensor_tma_kernel<Tag>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  launch_pdl(kern, dim3((unsigned)grid), dim3(kThreads), smem, st, static_cast<const uint8_t *>(x), head, body_bytes,
             tail, n, tiles, tile_bytes, stages, reinterpret_cast<uint32_t *>(slot));
  return check_launch("amax_tensor_tma_kernel");
}

template <typename Tag>
static int launch_amax_tensor(const void *x, size_t n, float *slot, cudaStream_t st) {
  if (n == 0) return B200Q_OK;
  if (tuning("amax_tma", 0) == 1 && reinterpret_cast<uintptr_t>(x) % Elem<Tag>::SIZE == 0)
    return launch_amax_tensor_tma<Tag>(x, n, slot, st);
  const int vb = tuning("vec_bytes", 32);
  const int unroll = tuning("amax_unroll", 4);
  const int ctas_per_sm = tuning("amax_ctas_per_sm", 0);  // 0: one tile per CTA
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
  B200Q_REQUIRE(addr % Elem<Tag>::SIZE == 0, "x is not element-aligned");
  size_t head = ((size_t)vb - addr % vb) % vb / Elem<Tag>::SIZE;
  if (head > n) head = n;
  const size_t epv = vb / Elem<Tag>::SIZE;
  const size_t nvec = (n - head) / epv;
  const size_t tail = n - head - nvec * epv;
  size_t tiles = (nvec + (size_t)kThreads * unroll - 1) / ((size_t)kThreads * unroll);
  if (tiles == 0) tiles = 1;
  size_t grid = tiles;
  if (ctas_per_sm > 0) grid = tiles < (size_t)sm_count() * ctas_per_sm ? tiles : (size_t)sm_count() * ctas_per_sm;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  uint32_t *sl = reinterpret_cast<uint32_t *>(slot);
#define LAUNCH(VB_, U_)                                                                            \
  launch_pdl(amax_tensor_kernel<Tag, VB_, U_>, dim3((unsigned)grid), dim3(kThreads), 0, st, xb, head, nvec, tail, tiles, sl)
  if (vb == 32) {
    if (unroll == 1) LAUNCH(32, 1);
    else if (unroll == 2) LAUNCH(32, 2);
    else if (unroll == 8) LAUNCH(32, 8);
    else LAUNCH(32, 4);
  } else {
    if (unroll == 1) LAUNCH(16, 1);
    else if (unroll == 2) LAUNCH(16, 2);
    else if (unroll == 8) LAUNCH(16, 8);
    else LAUNCH(16, 4);
  }
#undef LAUNCH
  return check_launch("amax_tensor_kernel");
}

// ---------------------------------------------------------------------------------------------
// per-row (segmented): rows of V vectors, L lanes per row
// ---------------------------------------------------------------------------------------------
template <typename Tag, int VB, int L>
__global__ void __launch_bounds__(kThreads)
    amax_rows_kernel(const Vec<VB> *__restrict__ xv, size_t n_rows, size_t V, size_t n_channels,
                     uint32_t *__restrict__ slots) {
  constexpr int ROWS_PER_WARP = 32 / L;
  const int lane = threadIdx.x & 31;
  const int sub = lane / L;     // which row of the warp's group
  const int lig = lane % L;     // lane within the row's group
  const size_t warp_global = (size_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  const size_t total_warps = (size_t)gridDim.x * (kThreads / 32);
  const size_t n_groups = (n_rows + ROWS_PER_WARP - 1) / ROWS_PER_WARP;
  const bool direct = (n_channels == n_rows);

  for (size_t g = warp_global; g < n_groups; g += total_warps) {
    const size_t row = g * ROWS_PER_WARP + sub;
    uint32_t acc = 0;
    if (row < n_rows) {
      const Vec<VB> *rp = xv + row * V;
      size_t v = lig;
      // 4 independent loads in flight per lane
      for (; v + 3 * (size_t)L < V; v += 4 * (size_t)L) {
        Vec<VB> a = ldg_stream(rp + v), b = ldg_stream(rp + v + L), c = ldg_stream(rp + v + 2 * L),
                d = ldg_stream(rp + v + 3 * L);
#pragma unroll
        for (int w = 0; w < Vec<VB>::WORDS; ++w) {
          acc = absmax_acc<Tag>(acc, a.r[w]);
          acc = absmax_acc<Tag>(acc, b.r[w]);
          acc = absmax_acc<Tag>(acc, c.r[w]);
          acc = absmax_acc<Tag>(acc, d.r[w]);
        }
      }
      for (; v < V; v += L) {
        Vec<VB> a = ldg_stream(rp + v);
#pragma unroll
        for (int w = 0; w < Vec<VB>::WORDS; ++w) acc = absmax_acc<Tag>(acc, a.r[w]);
      }
    }
    uint32_t m = group_max<L>(absmax_collapse<Tag>(acc));
    if (row < n_rows && lig == 0) {
      const uint32_t fb = Elem<Tag>::absbits_to_f32bits(m);
      if (direct) {
        const uint32_t old = slots[row];
        if (fb > old) slots[row] = fb;
      } else if (m != 0u) {
        atomicMax(slots + row % n_channels, fb);
      }
    }
  }
}

// long rows (>= one vector per thread): a CTA takes FOUR rows at once so that every thread has four
// independent 32-byte loads in flight, like the per-tensor kernel, and reduces them with one barrier.
template <typename Tag, int VB>
__global__ void __launch_bounds__(kThreads)
    amax_longrows_kernel(const Vec<VB> *__restrict__ xv, size_t n_rows, size_t V, size_t n_channels,
                         uint32_t *__restrict__ slots) {
  constexpr int R = 4;
  pdl_launch_dependents();
  pdl_wait();
  const size_t row0 = (size_t)blockIdx.x * R;
  uint32_t acc[R] = {0u, 0u, 0u, 0u};
  for (size_t v = threadIdx.x; v < V; v += kThreads) {
    Vec<VB> a[R];
#pragma unroll
    for (int k = 0; k < R; ++k) {
      if (row0 + k < n_rows) a[k] = ldg_stream(xv + (row0 + k) * V + v);
      else {
#pragma unroll
        for (int w = 0; w < Vec<VB>::WORDS; ++w) a[k].r[w] = 0u;
      }
    }
#pragma unroll
    for (int k = 0; k < R; ++k)
#pragma unroll
      for (int w = 0; w < Vec<VB>::WORDS; ++w) acc[k] = absmax_acc<Tag>(acc[k], a[k].r[w]);
  }
  __shared__ uint32_t s_part[R][kThreads / 32];
#pragma unroll
  for (int k = 0; k < R; ++k) {
    const uint32_t m = __reduce_max_sync(0xffffffffu, absmax_collapse<Tag>(acc[k]));
    if ((threadIdx.x & 31) == 0) s_part[k][threadIdx.x >> 5] = m;
  }
  __syncthreads();
  if (threadIdx.x < R && row0 + threadIdx.x < n_rows) {
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) m = max(m, s_part[threadIdx.x][w]);
    const size_t row = row0 + threadIdx.x;
    const uint32_t fb = Elem<Tag>::absbits_to_f32bits(m);
    if (n_channels == n_rows) {
      if (fb > slots[row]) slots[row] = fb;
    } else if (fb != 0u) {
      atomicMax(slots + row % n_channels, fb);
    }
  }
}

// rows that are exactly ONE vector long (NVFP4 block-16 amax of bf16 data with 32-byte vectors):
// one thread per row, 4 rows in flight per thread, slots read up front and written back once.
template <typename Tag, int VB>
__global__ void __launch_bounds__(kThreads)
    amax_vecrows_kernel(const Vec<VB> *__restrict__ xv, size_t n_rows, size_t n_channels,
                        uint32_t *__restrict__ slots) {
  constexpr int U = 4;
  pdl_launch_dependents();
  pdl_wait();
  const size_t base = (size_t)blockIdx.x * (kThreads * U) + threadIdx.x;
  const bool direct = (n_channels == n_rows);
  Vec<VB> v[U];
  uint32_t old[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const size_t r = base + (size_t)u * kThreads;
    old[u] = 0;
    if (r < n_rows) {
      v[u] = ldg_stream(xv + r);
      if (direct) old[u] = slots[r];
    }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const size_t r = base + (size_t)u * kThreads;
    if (r >= n_rows) continue;
    uint32_t acc = 0;
#pragma unroll
    for (int w = 0; w < Vec<VB>::WORDS; ++w) acc = absmax_acc<Tag>(acc, v[u].r[w]);
    const uint32_t fb = Elem<Tag>::absbits_to_f32bits(absmax_collapse<Tag>(acc));
    if (direct) {
      if (fb > old[u]) slots[r] = fb;
    } else if (fb != 0u) {
      atomicMax(slots + r % n_channels, fb);
    }
  }
}

// generic fallback: rows whose length / base is not vector aligned.  One warp per row, scalar.
template <typename Tag>
__global__ void __launch_bounds__(kThreads)
    amax_rows_scalar_kernel(const void *__restrict__ x, size_t n_rows, size_t row_len,
                            size_t n_channels, uint32_t *__restrict__ slots) {
  const int lane = threadIdx.x & 31;
  const size_t warp_global = (size_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  const size_t total_warps = (size_t)gridDim.x * (kThreads / 32);
  const uint32_t one_mask = Elem<Tag>::SIZE == 2 ? 0x7fffu : 0x7fffffffu;
  for (size_t row = warp_global; row < n_rows; row += total_warps) {
    uint32_t m = 0;
    for (size_t j = lane; j < row_len; j += 32) {
      uint32_t b;
      if constexpr (Elem<Tag>::SIZE == 2)
        b = reinterpret_cast<const uint16_t *>(x)[row * row_len + j];
      else
        b = reinterpret_cast<const uint32_t *>(x)[row * row_len + j];
      m = max(m, b & one_mask);
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if (lane == 0 && m != 0u) atomicMax(slots + row % n_channels, Elem<Tag>::absbits_to_f32bits(m));
  }
}

template <typename Tag, int VB>
static int launch_amax_rows_vb(const void *x, size_t n_rows, size_t V, size_t n_channels,
                               float *slots, cudaStream_t st) {
  const Vec<VB> *xv = static_cast<const Vec<VB> *>(x);
  uint32_t *sl = reinterpret_cast<uint32_t *>(slots);
  if (V >= (size_t)kThreads) {
    const size_t gridl = (n_rows + 3) / 4;
    B200Q_REQUIRE(gridl <= 0x7fffffffu, "tensor too large");
    launch_pdl(amax_longrows_kernel<Tag, VB>, dim3((unsigned)gridl), dim3(kThreads), 0, st, xv, n_rows, V, n_channels, sl);
    return check_launch("amax_longrows_kernel");
  }
  if (V == 1) {
    const size_t grid1 = (n_rows + (size_t)kThreads * 4 - 1) / ((size_t)kThreads * 4);
    B200Q_REQUIRE(grid1 <= 0x7fffffffu, "tensor too large");
    launch_pdl(amax_vecrows_kernel<Tag, VB>, dim3((unsigned)grid1), dim3(kThreads), 0, st, xv, n_rows, n_channels, sl);
    return check_launch("amax_vecrows_kernel");
  }
  int L = 1;
  while (L < 32 && (size_t)L < V) L <<= 1;  // smallest power of two >= V, capped at 32
  const size_t rows_per_warp = 32 / L;
  const size_t n_groups = (n_rows + rows_per_warp - 1) / rows_per_warp;
  const size_t warps_per_cta = kThreads / 32;
  size_t grid = (n_groups + warps_per_cta - 1) / warps_per_cta;
  // short rows: let every warp take a few row groups so enough loads are in flight
  const size_t cap = (size_t)sm_count() * 8 * (V <= (size_t)L ? 4 : 64);
  if (grid > cap) grid = cap;
  if (grid == 0) grid = 1;
#define LAUNCH(L_)                                                                                 \
  amax_rows_kernel<Tag, VB, L_><<<(unsigned)grid, kThreads, 0, st>>>(xv, n_rows, V, n_channels, sl)
  switch (L) {
  case 1: LAUNCH(1); break;
  case 2: LAUNCH(2); break;
  case 4: LAUNCH(4); break;
  case 8: LAUNCH(8); break;
  case 16: LAUNCH(16); break;
  default: LAUNCH(32); break;
  }
#undef LAUNCH
  return check_launch("amax_rows_kernel");
}

template <typename Tag>
static int launch_amax_rows(const void *x, size_t n_rows, size_t row_len, size_t n_channels,
                            float *slots, cudaStream_t st) {
  if (n_rows == 0 || row_len == 0) return B200Q_OK;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
  const size_t row_bytes = row_len * Elem<Tag>::SIZE;
  if (addr % 32 == 0 && row_bytes % 32 == 0 && tuning("vec_bytes", 32) == 32)
    return launch_amax_rows_vb<Tag, 32>(x, n_rows, row_bytes / 32, n_channels, slots, st);
  if (addr % 16 == 0 && row_bytes % 16 == 0)
    return launch_amax_rows_vb<Tag, 16>(x, n_rows, row_bytes / 16, n_channels, slots, st);
  B200Q_REQUIRE(addr % Elem<Tag>::SIZE == 0, "x is not element-aligned");
  size_t grid = (n_rows + kThreads / 32 - 1) / (kThreads / 32);
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
  amax_rows_scalar_kernel<Tag><<<(unsigned)grid, kThreads, 0, st>>>(
      x, n_rows, row_len, n_channels, reinterpret_cast<uint32_t *>(slots));
  return check_launch("amax_rows_scalar_kernel");
}

// ---------------------------------------------------------------------------------------------
// per-column: x [R, C]; a CTA owns a (32 lanes x VB) wide column strip and ROWS_PER_CTA rows.
// MODE 0: |x| max into u32 bit slots; MODE 1: sum |x| into fp32 slots.
// ---------------------------------------------------------------------------------------------
template <typename Tag, int VB, int MODE>
__global__ void __launch_bounds__(kThreads)
    cols_reduce_kernel(const uint8_t *__restrict__ x, size_t n_rows, size_t n_cols,
                       size_t rows_per_cta, void *__restrict__ slots) {
  constexpr int EPV = VB / Elem<Tag>::SIZE;
  constexpr int WARPS = kThreads / 32;
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t col0 = ((size_t)blockIdx.x * 32 + lane) * EPV;  // first column of this lane
  const size_t r_begin = (size_t)blockIdx.y * rows_per_cta;
  size_t r_end = r_begin + rows_per_cta;
  if (r_end > n_rows) r_end = n_rows;
  const bool active = col0 < n_cols;  // n_cols % EPV == 0 is guaranteed by the launcher

  uint32_t macc[Vec<VB>::WORDS];
  float sacc[EPV];
#pragma unroll
  for (int w = 0; w < Vec<VB>::WORDS; ++w) macc[w] = 0u;
#pragma unroll
  for (int e = 0; e < EPV; ++e) sacc[e] = 0.f;

  if (active) {
    const size_t row_bytes = n_cols * Elem<Tag>::SIZE;
    const uint8_t *p = x + col0 * Elem<Tag>::SIZE;
    auto fold = [&](const Vec<VB> &a) {
      if constexpr (MODE == 0) {
#pragma unroll
        for (int w = 0; w < Vec<VB>::WORDS; ++w) macc[w] = absmax_acc<Tag>(macc[w], a.r[w]);
      } else {
        float fa[EPV];
        vec_to_floats<Tag, VB>(a, fa);
#pragma unroll
        for (int e = 0; e < EPV; ++e) sacc[e] += fabsf(fa[e]);
      }
    };
    size_t r = r_begin + warp;
    for (; r + 3 * WARPS < r_end; r += 4 * WARPS) {  // four rows in flight per warp
      Vec<VB> a = ldg_stream(reinterpret_cast<const Vec<VB> *>(p + r * row_bytes));
      Vec<VB> b = ldg_stream(reinterpret_cast<const Vec<VB> *>(p + (r + WARPS) * row_bytes));
      Vec<VB> c = ldg_stream(reinterpret_cast<const Vec<VB> *>(p + (r + 2 * WARPS) * row_bytes));
      Vec<VB> d = ldg_stream(reinterpret_cast<const Vec<VB> *>(p + (r + 3 * WARPS) * row_bytes));
      fold(a);
      fold(b);
      fold(c);
      fold(d);
    }
    for (; r < r_end; r += WARPS) fold(ldg_stream(reinterpret_cast<const Vec<VB> *>(p + r * row_bytes)));
  }

  // combine the WARPS partials of each column through shared memory
  __shared__ uint32_t s_buf[WARPS][32][EPV + 1];
#pragma unroll
  for (int e = 0; e < EPV; ++e) {
    uint32_t val;
    if constexpr (MODE == 0) {
      if constexpr (Elem<Tag>::PER_WORD == 2)
        val = (e & 1) ? (macc[e / 2] >> 16) : (macc[e / 2] & 0xffffu);
      else
        val = macc[e];
    } else {
      val = __float_as_uint(sacc[e]);
    }
    s_buf[warp][lane][e] = val;
  }
  __syncthreads();
  // thread t handles column-in-strip t (32*EPV columns per strip; EPV <= 16 -> <= 512 columns)
  for (int c = threadIdx.x; c < 32 * EPV; c += kThreads) {
    const int ln = c / EPV, e = c % EPV;
    const size_t col = ((size_t)blockIdx.x * 32 + ln) * EPV + e;
    if (col >= n_cols) continue;
    if constexpr (MODE == 0) {
      uint32_t m = 0;
#pragma unroll
      for (int w = 0; w < WARPS; ++w) m = max(m, s_buf[w][ln][e]);
      if (m != 0u)
        atomicMax(reinterpret_cast<uint32_t *>(slots) + col, Elem<Tag>::absbits_to_f32bits(m));
    } else {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < WARPS; ++w) s += __uint_as_float(s_buf[w][ln][e]);
      atomicAdd(reinterpret_cast<float *>(slots) + col, s);
    }
  }
}

// scalar fallback for odd column counts / alignment
template <typename Tag, int MODE>
__global__ void __launch_bounds__(kThreads)
    cols_reduce_scalar_kernel(const void *__restrict__ x, size_t n_rows, size_t n_cols,
                              size_t rows_per_cta, void *__restrict__ slots) {
  const size_t col = (size_t)blockIdx.x * kThreads + threadIdx.x;
  if (col >= n_cols) return;
  const size_t r_begin = (size_t)blockIdx.y * rows_per_cta;
  size_t r_end = r_begin + rows_per_cta;
  if (r_end > n_rows) r_end = n_rows;
  float s = 0.f, m = 0.f;
  bool nan = false;
  for (size_t r = r_begin; r < r_end; ++r) {
    const float v = fabsf(Elem<Tag>::load1(x, r * n_cols + col));
    if (v != v) nan = true;
    m = fmaxf(m, v);
    s += v;
  }
  if constexpr (MODE == 0) {
    uint32_t b = nan ? 0x7fc00000u : __float_as_uint(m);
    if (b != 0u) atomicMax(reinterpret_cast<uint32_t *>(slots) + col, b);
  } else {
    atomicAdd(reinterpret_cast<float *>(slots) + col, s);
  }
}

template <typename Tag, int MODE>
static int launch_cols(const void *x, size_t n_rows, size_t n_cols, void *slots, cudaStream_t st) {
  if (n_rows == 0 || n_cols == 0) return B200Q_OK;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
  const size_t row_bytes = n_cols * Elem<Tag>::SIZE;
  // rows per CTA: enough CTAs to fill the chip ~4x over, at least 16 rows each
  auto rows_per_cta_for = [&](size_t strips) {
    // ~4 CTAs per SM; whole multiples of the 32-row unrolled step so the 4-loads-in-flight loop covers
    // the chunk, and few enough chunks that the per-column atomics (one per CTA per column) stay cheap
    size_t want_ctas = (size_t)sm_count() * 4;
    size_t chunks = (want_ctas + strips - 1) / strips;
    if (chunks < 1) chunks = 1;
    size_t rpc = (n_rows + chunks - 1) / chunks;
    rpc = (rpc + 31) / 32 * 32;
    if (rpc < 32) rpc = 32;
    return rpc;
  };
  auto launch_vec = [&](auto vb_tag) -> int {
    constexpr int VB = decltype(vb_tag)::value;
    constexpr int EPV = VB / Elem<Tag>::SIZE;
    const size_t strips = (n_cols / EPV + 31) / 32;
    const size_t rpc = rows_per_cta_for(strips);
    const size_t chunks = (n_rows + rpc - 1) / rpc;
    B200Q_REQUIRE(chunks <= 65535, "too many row chunks");
    dim3 grid((unsigned)strips, (unsigned)chunks);
    launch_pdl(cols_reduce_kernel<Tag, VB, MODE>, grid, dim3(kThreads), 0, st, static_cast<const uint8_t *>(x), n_rows,
               n_cols, rpc, slots);
    return check_launch("cols_reduce_kernel");
  };
  if (addr % 32 == 0 && row_bytes % 32 == 0 && n_cols >= 2048 && tuning("vec_bytes", 32) == 32)
    return launch_vec(std::integral_constant<int, 32>{});
  if (addr % 16 == 0 && row_bytes % 16 == 0) return launch_vec(std::integral_constant<int, 16>{});
  B200Q_REQUIRE(addr % Elem<Tag>::SIZE == 0, "x is not element-aligned");
  const size_t strips = (n_cols + kThreads - 1) / kThreads;
  const size_t rpc = rows_per_cta_for(strips);
  const size_t chunks = (n_rows + rpc - 1) / rpc;
  B200Q_REQUIRE(chunks <= 65535, "too many row chunks");
  dim3 grid((unsigned)strips, (unsigned)chunks);
  cols_reduce_scalar_kernel<Tag, MODE><<<grid, kThreads, 0, st>>>(x, n_rows, n_cols, rpc, slots);
  return check_launch("cols_reduce_scalar_kernel");
}

// ---------------------------------------------------------------------------------------------
// export
// ---------------------------------------------------------------------------------------------
__global__ void amax_export_kernel(const float *__restrict__ slots, size_t n, void *dst, int dt) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = slots[i];
  if (dt == B200Q_F32) ((float *)dst)[i] = v;
  else if (dt == B200Q_BF16) ((uint16_t *)dst)[i] = f2bf_bits(v);
  else ((uint16_t *)dst)[i] = f2h_bits(v);
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_amax_per_tensor_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, float *slots,
                                b200q_stream_t stream) {
  if (n_desc == 0 || total_ctas == 0) return B200Q_OK;
  B200Q_REQUIRE(descs != nullptr && slots != nullptr && n_desc > 0, "null pointer");
  B200Q_REQUIRE(total_ctas <= 0x7fffffffu, "too many CTAs");
  const MultiDesc *d = static_cast<const MultiDesc *>(descs);
  uint32_t *sl = reinterpret_cast<uint32_t *>(slots);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       launch_pdl(amax_tensor_multi_kernel<Tag, 32, 4>, dim3((unsigned)total_ctas), dim3(kThreads), 0,
                                  (cudaStream_t)stream, d, n_desc, sl));
  return check_launch("amax_tensor_multi_kernel");
}

int b200q_amax_per_tensor(const void *x, int dtype, size_t n, float *amax_slot,
                          b200q_stream_t stream) {
  B200Q_REQUIRE(amax_slot != nullptr, "amax_slot is null");
  B200Q_REQUIRE(x != nullptr || n == 0, "x is null");
  B200Q_DISPATCH_DTYPE(dtype, Tag, return launch_amax_tensor<Tag>(x, n, amax_slot, (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_amax_rows(const void *x, int dtype, size_t n_rows, size_t row_len, size_t n_channels,
                    float *amax_slots, b200q_stream_t stream) {
  B200Q_REQUIRE(amax_slots != nullptr, "amax_slots is null");
  B200Q_REQUIRE(x != nullptr || n_rows * row_len == 0, "x is null");
  B200Q_REQUIRE(n_channels > 0 && n_channels <= (n_rows ? n_rows : 1), "bad n_channels");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_amax_rows<Tag>(x, n_rows, row_len, n_channels, amax_slots,
                                                    (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_amax_cols(const void *x, int dtype, size_t n_rows, size_t n_cols, float *amax_slots,
                    b200q_stream_t stream) {
  B200Q_REQUIRE(amax_slots != nullptr, "amax_slots is null");
  B200Q_REQUIRE(x != nullptr || n_rows * n_cols == 0, "x is null");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return (launch_cols<Tag, 0>(x, n_rows, n_cols, amax_slots, (cudaStream_t)stream)));
  return B200Q_OK;
}

int b200q_abssum_cols(const void *x, int dtype, size_t n_rows, size_t n_cols, float *sum_slots,
                      b200q_stream_t stream) {
  B200Q_REQUIRE(sum_slots != nullptr, "sum_slots is null");
  B200Q_REQUIRE(x != nullptr || n_rows * n_cols == 0, "x is null");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return (launch_cols<Tag, 1>(x, n_rows, n_cols, sum_slots, (cudaStream_t)stream)));
  return B200Q_OK;
}

int b200q_amax_export(const float *amax_slots, size_t n, void *dst, int dtype,
                      b200q_stream_t stream) {
  B200Q_REQUIRE(amax_slots != nullptr && dst != nullptr, "null pointer");
  B200Q_REQUIRE(dtype_ok(dtype), "unknown dtype %d", dtype);
  if (n == 0) return B200Q_OK;
  amax_export_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(amax_slots, n,
                                                                                  dst, dtype);
  return check_launch("amax_export_kernel");
}

}  // extern "C"
