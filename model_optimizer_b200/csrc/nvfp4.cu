// nvfp4.cu -- NVFP4 (E2M1 values, E4M3 scale per 16-element block, fp32 per-tensor scale):
// dynamic / static fake quant, quant-and-pack, unpack.
//
// One thread owns one 16-element block: one 32-byte vector (two LDG.E.128) brings the block into
// registers, the block amax is an in-register packed-integer max (no shuffles), the two-level
// scale is computed once per block, E2M1 rounding is the reference's round-to-nearest-even, branch-free
// (e2m1_round_mag / f32x2_to_e2m1x2 in common.cuh: sm_90 has no FP4 convert), and the block leaves with
// one 32-byte vector store (fake quant) or one 8-byte + one 1-byte store (pack).  The grouped dynamic fake quant
// (nvfp4_dyn_multi_kernel) instead maps each whole tile of a 16-bit tensor lane-contiguously, two lanes per block
// (dyn_fq_tile), so that every warp load and store fills whole 32-byte sectors.
//
// Reference semantics:
//   dynamic fake quant : kernels/quantization/gemm/fp4_kernel_hopper.py:33-170 +
//                        kernels/quantization/common/nvfp4_quant.py:33-126  (IEEE division here;
//                        the Triton kernel's approximate division only differs at exact ties)
//   static fake quant  : kernels/quantization/gemm/fp4_kernel.py:194-316
//   pack / unpack      : quantization/qtensor/nvfp4_tensor.py:32-48, 139-161, 204-342, 344-407
#include "block16.cuh"

namespace b200q {

constexpr int kNvThreads = 256;

// ---------------------------------------------------------------------------------------------
// dynamic fake quant
// ---------------------------------------------------------------------------------------------
// dynamic fake quant of the blocks base + u * stride (u < UNROLL) that are below n.  COLLECT: also returns their |x|
// max as raw magnitude bits in the element's own format -- what amax_tensor_multi_kernel reduces, NaN payload included
// (the block scale is the same either way: a non-finite block max gives the 448 clamp whatever its payload); 0 otherwise.
template <typename Tag, int VB, int UNROLL, bool COLLECT>
__device__ __forceinline__ uint32_t dyn_fq_blocks(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t base,
                                                  size_t stride, size_t n, const DynScale &ds, const ExactDiv &d6) {
  Block<Tag, VB> b[UNROLL];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * stride;
    if (i < n) b[u].load(x, i);
  }
  uint32_t amax = 0;
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * stride;
    if (i >= n) continue;
    uint32_t mb;
    if constexpr (COLLECT) {
      const uint32_t nb = b[u].prep_and_absmax_native_bits();
      amax = max(amax, nb);
      mb = Elem<Tag>::absbits_to_f32bits(nb);
    } else {
      mb = b[u].prep_and_absmax_bits();
    }
    const bool finite = mb < 0x7f800000u;
    const float s = ds.block_scale(dyn_block_max(b[u], mb), d6);
    qdq_block<Tag, VB>(b[u], s, finite);
    b[u].store(y, i);
  }
  return amax;
}

// dyn_fq_blocks over the whole tile of kNvThreads * UNROLL blocks from block `tile`, 16-bit types, lane-contiguous: warp
// w owns the tile's bytes [w, w + 1) * 32 * H * 16 and load i of lane l is the 16 bytes at i * 512 + l * 16 of them,
// so each warp instruction covers 512 contiguous bytes (16 whole 32-byte sectors) where dyn_fq_blocks' covers half
// of 32 sectors.  Lanes 2k and 2k + 1 hold the two halves of one block: each reduces its 8 elements, one shuffle
// gives both lanes the block's |x| max, and each quantizes and stores its own half.  Same bits as dyn_fq_blocks,
// and (COLLECT) the same CTA max of the returned values.
template <typename Tag, int UNROLL, bool COLLECT>
__device__ __forceinline__ uint32_t dyn_fq_tile(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t tile,
                                                const DynScale &ds, const ExactDiv &d6) {
  static_assert(Elem<Tag>::SIZE == 2, "a lane's 16 bytes are half a block only for 16-bit types");
  constexpr int H = 2 * UNROLL;  // half blocks per lane
  Block<Tag, 16, kBlk / 2> h[H];
  // in half blocks (16 bytes): the tile starts at 2 * tile, warp w's bytes at 32 * H * w
  const size_t h0 = 2 * tile + (size_t)(threadIdx.x >> 5) * (32 * H) + (threadIdx.x & 31);
#pragma unroll
  for (int i = 0; i < H; ++i) h[i].load(x, h0 + 32 * i);
  // The stores mark their L2 lines evict-first: nothing reads the output back within the pass, and on an H100 the
  // pass is 1.8 % faster than with default-priority stores (the hint on the loads made no difference; DESIGN §5).
  const uint64_t pol = l2_evict_first_policy();
  Vec<16> *dst = reinterpret_cast<Vec<16> *>(y) + h0;
  uint32_t amax = 0;
#pragma unroll
  for (int i = 0; i < H; ++i) {
    uint32_t mb;
    if constexpr (COLLECT) {
      const uint32_t nb = h[i].prep_and_absmax_native_bits();
      amax = max(amax, nb);
      mb = Elem<Tag>::absbits_to_f32bits(nb);
    } else {
      mb = h[i].prep_and_absmax_bits();
    }
    mb = max(mb, __shfl_xor_sync(0xffffffffu, mb, 1));
    const bool finite = mb < 0x7f800000u;
    const float s = ds.block_scale(dyn_pair_block_max(h[i], mb), d6);
    qdq_block(h[i], s, finite);
    stg(dst + 32 * i, h[i].v[0], pol);
  }
  return amax;
}

template <typename Tag, int VB, int UNROLL>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_dyn_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t n_blocks,
                     const void *__restrict__ gamax, int gamax_dtype) {
  pdl_launch_dependents();
  pdl_wait();
  DynScale ds;
  ds.setup(load_scalar(gamax, gamax_dtype, 0));
  const ExactDiv d6(ds.six_gs);
  const size_t base = (size_t)blockIdx.x * (kNvThreads * UNROLL) + threadIdx.x;
  dyn_fq_blocks<Tag, VB, UNROLL, false>(x, y, base, kNvThreads, n_blocks, ds, d6);
}

// TMA-store variant (north-star "TMA bulk staging" on the WRITE side; knob "nvfp4_tma_store"): the CTA's 16 KB of
// results are staged in shared memory and leave as ONE cp.async.bulk.global.shared::cta (UBLKCP) issued by an elected
// thread instead of 512 32-byte vector stores.  Bit-identical to the STG kernel.
template <typename Tag, int UNROLL>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_dyn_tma_store_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t n_blocks,
                               const void *__restrict__ gamax, int gamax_dtype) {
  constexpr int VB = 32;
  constexpr int BLOCK_BYTES = kBlk * Elem<Tag>::SIZE;                       // 32 (16-bit) or 64 (fp32)
  constexpr uint32_t TILE_BYTES = kNvThreads * UNROLL * BLOCK_BYTES;
  extern __shared__ __align__(128) uint8_t s_out[];
  pdl_launch_dependents();
  pdl_wait();
  DynScale ds;
  ds.setup(load_scalar(gamax, gamax_dtype, 0));
  const ExactDiv d6(ds.six_gs);
  const size_t tile0 = (size_t)blockIdx.x * (kNvThreads * UNROLL);          // first 16-block of this CTA's tile
  Block<Tag, VB> b[UNROLL];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) b[u].load(x, tile0 + (size_t)u * kNvThreads + threadIdx.x);
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const uint32_t mb = b[u].prep_and_absmax_bits();
    const bool finite = mb < 0x7f800000u;
    const float s = ds.block_scale(dyn_block_max(b[u], mb), d6);
    qdq_block<Tag, VB>(b[u], s, finite);
    Vec<VB> *sp = reinterpret_cast<Vec<VB> *>(s_out) + ((size_t)u * kNvThreads + threadIdx.x) * Block<Tag, VB>::NV;
#pragma unroll
    for (int i = 0; i < Block<Tag, VB>::NV; ++i) sp[i] = b[u].v[i];        // plain stores -> st.shared
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");              // make the writes visible to the async proxy
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t src = (uint32_t)__cvta_generic_to_shared(s_out);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(y + tile0 * BLOCK_BYTES), "r"(src),
                 "r"(TILE_BYTES)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");          // smem must outlive the read by the copy engine
  }
}

// nvfp4_dyn_kernel over a table of tensors (common.cuh MultiDesc): CTA -> (tensor, tile of 256 * UNROLL blocks);
// each tensor's global amax is amax_base[slot] (the engine's flat _amax arena).  A whole tile of a 16-bit tensor goes
// through dyn_fq_tile, the partial last tile of an entry (and every fp32 tile) through dyn_fq_blocks: the CTA owns the
// same bytes either way.
// COLLECT: the pass is also the calibration collect -- the CTA's |x| max goes into the fp32 slot slots[slot] exactly as
// amax_tensor_multi_kernel puts it there (unsigned atomic max on the bit pattern, nothing for an all-zero tile), so the
// slot ends bit-identical to that kernel's.  The atomic is skipped when the slot already holds at least that value:
// slots only grow, so the skip is exact.
template <typename Tag, int VB, int UNROLL, bool COLLECT>
__global__ void __launch_bounds__(kNvThreads, !COLLECT ? 0 : std::is_same<Tag, BF16Tag>::value ? 5 : 4)
    nvfp4_dyn_multi_kernel(const MultiDesc *__restrict__ descs, int n_desc, const void *__restrict__ amax_base,
                           int gamax_dtype, uint32_t *__restrict__ slots) {
  pdl_launch_dependents();
  pdl_wait();
  const MultiDesc d = descs[multi_find(descs, n_desc)];
  DynScale ds;
  ds.setup(load_scalar(amax_base, gamax_dtype, (size_t)d.slot));
  const ExactDiv d6(ds.six_gs);
  const size_t tile = (size_t)(blockIdx.x - d.first_cta) * (kNvThreads * UNROLL);
  uint32_t m = 0;
  if constexpr (Elem<Tag>::SIZE == 2) {  // fp32 (64-byte blocks) keeps the per-block mapping
    if (tile + kNvThreads * UNROLL <= d.n_units) {
      m = dyn_fq_tile<Tag, UNROLL, COLLECT>(d.x, d.y, tile, ds, d6);
    } else {  // the partial last tile of an entry, one block per thread at a time: no spills at 5 CTAs / SM
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
        m = max(m, dyn_fq_blocks<Tag, VB, 1, COLLECT>(d.x, d.y, tile + u * kNvThreads + threadIdx.x, kNvThreads,
                                                      d.n_units, ds, d6));
    }
  } else {
    m = dyn_fq_blocks<Tag, VB, UNROLL, COLLECT>(d.x, d.y, tile + threadIdx.x, kNvThreads, d.n_units, ds, d6);
  }
  if constexpr (COLLECT) {
    const uint32_t cm = block_max<kNvThreads>(m);
    if (threadIdx.x == 0 && cm != 0u) {
      const uint32_t fb = Elem<Tag>::absbits_to_f32bits(cm);
      if (fb > __ldcg(slots + d.slot)) atomicMax(slots + d.slot, fb);
    }
  }
}

// The amax the export is about to give entry e -- its fp32 slot rounded to amax_dtype as amax_export_kernel rounds
// it -- and whether it differs in bits from amax_base[slot] (what the speculative pass used).
__device__ __forceinline__ float exported_amax(const MultiDesc &d, const uint32_t *__restrict__ slots,
                                               const void *__restrict__ amax_base, int amax_dtype, bool &changed) {
  const long long slot = d.slot;
  const float v = __uint_as_float(__ldcg(slots + slot));
  uint32_t nb, ob;
  float na;
  if (amax_dtype == B200Q_F32) {
    nb = __float_as_uint(v);
    ob = static_cast<const uint32_t *>(amax_base)[slot];
    na = v;
  } else if (amax_dtype == B200Q_BF16) {
    nb = f2bf_bits(v);
    ob = static_cast<const uint16_t *>(amax_base)[slot];
    na = __uint_as_float(nb << 16);
  } else {
    nb = f2h_bits(v);
    ob = static_cast<const uint16_t *>(amax_base)[slot];
    na = h2f_bits((uint16_t)nb);
  }
  changed = nb != ob;
  return na;
}

// the whole CTA quantizes blocks [from, to) of entry d with amax a
template <typename Tag, int VB, int UNROLL>
__device__ __forceinline__ void cta_fq_range(const MultiDesc &d, size_t from, size_t to, float a) {
  DynScale ds;
  ds.setup(a);
  const ExactDiv d6(ds.six_gs);
  for (size_t i = from + threadIdx.x; i < to; i += (size_t)kNvThreads * UNROLL)
    dyn_fq_blocks<Tag, VB, UNROLL, false>(d.x, d.y, i, kNvThreads, to, ds, d6);
}

// Exact fix-up after a speculative COLLECT pass (which quantized with the amax exported one step earlier), two kinds
// of work over one persistent grid:
//  1. an entry whose exported amax changes (exported_amax) is quantized again with the new amax over its live blocks
//     [live_from, n_units) (live[2 i] = live_from, ops.live_block_ranges): the prefix below live_from is overwritten by
//     later entries of the table that share the output buffer, and the live ranges of different entries never
//     overlap.  Every CTA checks the entries 256 at a time (one per thread) and grid-strides over the range of each
//     changed one; redo_count gets one increment each.
//  2. pieces[3 p .. 3 p + 2] = (entry, from, to): the live blocks of the pre-flagged output tiles (ops.output_tiles),
//     where live blocks of two entries meet, so that neither pass of the fused step can order all their stores; one
//     CTA per piece.  It uses the exported amax too, so it writes what 1 writes where they meet.
// Every other live block was stored last by the second pass of the fused step, after the first pass had completed.
template <typename Tag, int VB, int UNROLL>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_dyn_multi_fixup_kernel(const MultiDesc *__restrict__ descs, const unsigned long long *__restrict__ live,
                                 int n_desc, const uint32_t *__restrict__ slots, const void *__restrict__ amax_base,
                                 int amax_dtype, const long long *__restrict__ pieces, int n_pieces,
                                 int *__restrict__ redo_count) {
  __shared__ uint32_t s_work[kNvThreads / 32];
  __shared__ float s_amax[kNvThreads];
  pdl_launch_dependents();
  pdl_wait();
  const size_t stride = (size_t)gridDim.x * kNvThreads;
  const size_t gtid = (size_t)blockIdx.x * kNvThreads + threadIdx.x;
  for (int e0 = 0; e0 < n_desc; e0 += kNvThreads) {
    const int e = e0 + (int)threadIdx.x;
    bool work = false;
    if (e < n_desc) {
      bool redo;
      s_amax[threadIdx.x] = exported_amax(descs[e], slots, amax_base, amax_dtype, redo);
      work = redo && descs[e].n_units > live[2 * e];
      if (redo && blockIdx.x == 0) atomicAdd(redo_count, 1);
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, work);
    if ((threadIdx.x & 31) == 0) s_work[threadIdx.x >> 5] = ballot;
    __syncthreads();
    for (int w = 0; w < kNvThreads / 32; ++w) {
      for (uint32_t bits = s_work[w]; bits != 0u; bits &= bits - 1u) {
        const int k = w * 32 + __ffs((int)bits) - 1;
        const MultiDesc d = descs[e0 + k];
        const size_t end = d.n_units;
        DynScale ds;
        ds.setup(s_amax[k]);
        const ExactDiv d6(ds.six_gs);
        for (size_t i = live[2 * (e0 + k)] + gtid; i < end; i += stride * UNROLL)
          dyn_fq_blocks<Tag, VB, UNROLL, false>(d.x, d.y, i, stride, end, ds, d6);
      }
    }
    __syncthreads();  // s_work / s_amax are refilled for the next 256 entries
  }
  for (int p = blockIdx.x; p < n_pieces; p += gridDim.x) {
    const MultiDesc d = descs[pieces[3 * p]];
    bool redo;
    const float a = exported_amax(d, slots, amax_base, amax_dtype, redo);
    cta_fq_range<Tag, VB, UNROLL>(d, (size_t)pieces[3 * p + 1], (size_t)pieces[3 * p + 2], a);
  }
}

template <typename Tag>
static int launch_nvfp4_fixup(const MultiDesc *d, const unsigned long long *live, int n_desc, const uint32_t *slots,
                              const void *amax_base, int amax_dtype, const long long *pieces, int n_pieces,
                              int *redo_count, cudaStream_t st) {
  auto kern = nvfp4_dyn_multi_fixup_kernel<Tag, 32, 2>;
  static int per_sm = 0;  // resident CTAs per SM: the grid is exactly one wave, so no CTA waits for another to finish
  if (per_sm == 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kNvThreads, 0) != cudaSuccess)
    return check_launch("nvfp4_dyn_multi_fixup_kernel occupancy");
  const int grid = sm_count() * (per_sm < 1 ? 1 : per_sm);
  launch_pdl(kern, dim3((unsigned)grid), dim3(kNvThreads), 0, st, d, live, n_desc, slots, amax_base, amax_dtype,
             pieces, n_pieces, redo_count);
  return check_launch("nvfp4_dyn_multi_fixup_kernel");
}

// ragged rows (row_len % 16 != 0) or unaligned tensors: one thread per (row, block), scalar I/O
template <typename Tag>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_dyn_ragged_kernel(const void *__restrict__ x, void *__restrict__ y, size_t n_rows,
                            size_t row_len, size_t blocks_per_row,
                            const void *__restrict__ gamax, int gamax_dtype) {
  DynScale ds;
  ds.setup(load_scalar(gamax, gamax_dtype, 0));
  const ExactDiv d6(ds.six_gs);
  const size_t total = n_rows * blocks_per_row;
  for (size_t t = blockIdx.x * (size_t)kNvThreads + threadIdx.x; t < total;
       t += (size_t)gridDim.x * kNvThreads) {
    const size_t row = t / blocks_per_row, bk = t % blocks_per_row;
    const size_t c0 = bk * kBlk;
    const int cnt = (int)((row_len - c0) < (size_t)kBlk ? (row_len - c0) : (size_t)kBlk);
    float f[kBlk];
    float bmax = __uint_as_float(0x7fc00000u);   // NaN-ignoring max, as dyn_block_max
    for (int e = 0; e < kBlk; ++e) {
      f[e] = e < cnt ? Elem<Tag>::load1(x, row * row_len + c0 + e) : 0.0f;
      bmax = fmaxf(bmax, fabsf(f[e]));
    }
    const float s = ds.block_scale(bmax, d6);
    for (int e = 0; e < cnt; ++e) {
      const float r = __fmul_rn(e2m1_round_mag(__fdiv_rn(fabsf(f[e]), s)), s);
      Elem<Tag>::store1(y, row * row_len + c0 + e, (f[e] >= 0.f) ? r : -r);
    }
  }
}


template <typename Tag>
static int launch_nvfp4_dyn(const void *x, void *y, size_t n_rows, size_t row_len,
                            const void *gamax, int gamax_dtype, cudaStream_t st) {
  const size_t n = n_rows * row_len;
  if (n == 0) return B200Q_OK;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), ay = reinterpret_cast<uintptr_t>(y);
  B200Q_REQUIRE(ax % Elem<Tag>::SIZE == 0 && ay % Elem<Tag>::SIZE == 0, "tensor not element-aligned");
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  uint8_t *yb = static_cast<uint8_t *>(y);
  if (row_len % kBlk == 0 && ax % 16 == 0 && ay % 16 == 0) {
    const size_t n_blocks = n / kBlk;
    const int unroll = tuning("nvfp4_unroll", 2);
    const bool v32 = (ax % 32 == 0) && (ay % 32 == 0) && tuning("vec_bytes", 32) == 32;
    const size_t per_cta = (size_t)kNvThreads * unroll;
    const size_t grid = (n_blocks + per_cta - 1) / per_cta;
    B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
    if (tuning("nvfp4_tma_store", 0) == 1 && v32 && n_blocks % (kNvThreads * 2) == 0) {
      const size_t smem = (size_t)kNvThreads * 2 * kBlk * Elem<Tag>::SIZE;
      launch_pdl(nvfp4_dyn_tma_store_kernel<Tag, 2>, dim3((unsigned)(n_blocks / (kNvThreads * 2))), dim3(kNvThreads), smem,
                 st, xb, yb, n_blocks, gamax, gamax_dtype);
      return check_launch("nvfp4_dyn_tma_store_kernel");
    }
#define LAUNCH(VB_, U_)                                                                            \
  launch_pdl(nvfp4_dyn_kernel<Tag, VB_, U_>, dim3((unsigned)grid), dim3(kNvThreads), 0, st, xb, yb, n_blocks, gamax, gamax_dtype)
    if (v32) {
      if (unroll == 1) LAUNCH(32, 1);
      else if (unroll == 4) LAUNCH(32, 4);
      else LAUNCH(32, 2);
    } else {
      if (unroll == 1) LAUNCH(16, 1);
      else if (unroll == 4) LAUNCH(16, 4);
      else LAUNCH(16, 2);
    }
#undef LAUNCH
    return check_launch("nvfp4_dyn_kernel");
  }
  const size_t bpr = (row_len + kBlk - 1) / kBlk;
  size_t grid = (n_rows * bpr + kNvThreads - 1) / kNvThreads;
  const size_t cap = (size_t)sm_count() * 32;
  if (grid > cap) grid = cap;
  nvfp4_dyn_ragged_kernel<Tag><<<(unsigned)grid, kNvThreads, 0, st>>>(x, y, n_rows, row_len, bpr, gamax, gamax_dtype);
  return check_launch("nvfp4_dyn_ragged_kernel");
}

// ---------------------------------------------------------------------------------------------
// static fake quant: calibrated per-block amax (fp4_kernel.py:217-316)
// ---------------------------------------------------------------------------------------------
template <typename Tag, int VB, int UNROLL>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_static_kernel(const uint8_t *__restrict__ x, uint8_t *__restrict__ y, size_t n_blocks,
                        const float *__restrict__ block_amax, const float *__restrict__ global_amax,
                        int quantize, float ratio) {
  pdl_launch_dependents();
  pdl_wait();
  StaticScale ss;
  ss.setup(global_amax, quantize, ratio);
  const size_t base = (size_t)blockIdx.x * (kNvThreads * UNROLL) + threadIdx.x;
  Block<Tag, VB> b[UNROLL];
  float am[UNROLL];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * kNvThreads;
    if (i < n_blocks) {
      b[u].load(x, i);
      am[u] = block_amax[i];
    }
  }
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * kNvThreads;
    if (i >= n_blocks) continue;
    const uint32_t mb = b[u].prep_and_absmax_bits();
    const bool finite = mb < 0x7f800000u;
    static_qdq_block<Tag, VB>(b[u], ss.block_scale(am[u]), finite);
    b[u].store(y, i);
  }
}

template <typename Tag>
static int launch_nvfp4_static(const void *x, void *y, size_t n_blocks, const float *block_amax,
                               const float *global_amax, int quantize, float fp8_max_norm,
                               cudaStream_t st) {
  if (n_blocks == 0) return B200Q_OK;
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x), ay = reinterpret_cast<uintptr_t>(y);
  B200Q_REQUIRE(ax % 16 == 0 && ay % 16 == 0, "static NVFP4 fake quant needs 16-byte aligned tensors");
  const float ratio = (float)(448.0 / (double)fp8_max_norm);
  const int unroll = tuning("nvfp4_unroll", 2);
  const bool v32 = (ax % 32 == 0) && (ay % 32 == 0) && tuning("vec_bytes", 32) == 32;
  const size_t per_cta = (size_t)kNvThreads * unroll;
  const size_t grid = (n_blocks + per_cta - 1) / per_cta;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  uint8_t *yb = static_cast<uint8_t *>(y);
#define LAUNCH(VB_, U_)                                                                            \
  launch_pdl(nvfp4_static_kernel<Tag, VB_, U_>, dim3((unsigned)grid), dim3(kNvThreads), 0, st, xb, yb, n_blocks, block_amax, global_amax, quantize, ratio)
  if (v32) {
    if (unroll == 1) LAUNCH(32, 1);
    else if (unroll == 4) LAUNCH(32, 4);
    else LAUNCH(32, 2);
  } else {
    if (unroll == 1) LAUNCH(16, 1);
    else if (unroll == 4) LAUNCH(16, 4);
    else LAUNCH(16, 2);
  }
#undef LAUNCH
  return check_launch("nvfp4_static_kernel");
}

// ---------------------------------------------------------------------------------------------
// quant-and-pack (NVFP4QTensor.quantize, nvfp4_tensor.py:229-342)
// ---------------------------------------------------------------------------------------------
// _cast_fp4 of one quotient pair on the slow path (nvfp4_tensor.py:229-251): sign from (y < 0) only,
// NaN -> ordinal 7.  Out of line: it only runs for non-finite blocks / scales outside the window.
__device__ __noinline__ uint32_t encode_pair_slow(float x0, float x1, float denom) {
  const float a0 = __fdiv_rn(x0, denom), a1 = __fdiv_rn(x1, denom);
  const uint32_t c = f32x2_to_e2m1x2(a0, a1) & 0xffu;
  const uint32_t c0 = (a0 != a0) ? 7u : ((c & 0x7u) | ((a0 < 0.f) ? 8u : 0u));
  const uint32_t c1 = (a1 != a1) ? 7u : (((c >> 4) & 0x7u) | ((a1 < 0.f) ? 8u : 0u));
  return c0 | (c1 << 4);
}

// codes for the 16 elements of a block given the combined divisor denom = float(bs8) * s2; amax_b: the quant block's
// |x| max (+inf / NaN for a non-finite block)
template <typename Tag, int VB>
__device__ __forceinline__ uint2 encode_block(Block<Tag, VB> &b, float denom, float amax_b) {
  float f[kBlk];
  b.to_floats(f);
  uint32_t lo = 0, hi = 0;
  const ExactDiv d(denom);
  // upper bound of the window: the smallest non-zero |x| of the element type (2^-133 bf16, 2^-24 fp16, 2^-149 fp32)
  // divided by denom must not round to zero -- a quotient that underflows to -0.0 loses the sign below, while the
  // reference's (-0.0 < 0) is false; such blocks take the explicit path
  constexpr float kMaxDenom = std::is_same<Tag, BF16Tag>::value ? 0x1p16f : (std::is_same<Tag, F16Tag>::value ? 0x1p60f : 1.0f);
  // and no quotient may overflow: for x = -1e30 and denom = 5e-10, q = x * y = -inf, the residual is +inf and the
  // correction fma(y, +inf, -inf) is NaN -- a code without x's sign, where the reference's -inf gives 0xF.  With
  // |x| <= 2^126 * denom every q is finite (any |q| > 5 is code 7 whatever its last bits).  2^126 * denom is exact for
  // denom in the window or overflows, hence the FLT_MAX cap: it keeps inf / NaN blocks on the explicit path
  const bool fast = d.block_ok(amax_b <= fminf(__fmul_rn(0x1p126f, denom), 0x1.fffffep127f), kMaxDenom);
  if (fast) {
    // the correctly rounded quotient carries the sign the reference derives from (weight < 0): q = x * y has x's sign,
    // the residual only corrects its last bit, and for x = -0.0 the chain gives (+0) + (-0) = +0 -- sign bit clear,
    // exactly as (-0.0 < 0) is false.  So no sign fix-up and no -0.0 normalisation of the inputs is needed here.
#pragma unroll
    for (int e = 0; e < kBlk; e += 2) {
      float a0 = f[e], a1 = f[e + 1];
      d.quot2(a0, a1);
      const uint32_t c = f32x2_to_e2m1x2(a0, a1) & 0xffu;  // byte = code[odd] << 4 | code[even]
      if (e < 8) lo |= c << (4 * e);
      else hi |= c << (4 * (e - 8));
    }
  } else {
#pragma unroll
    for (int e = 0; e < kBlk; e += 2) {
      const uint32_t c = encode_pair_slow(f[e], f[e + 1], denom);
      if (e < 8) lo |= c << (4 * e);
      else hi |= c << (4 * (e - 8));
    }
  }
  return make_uint2(lo, hi);
}

template <typename Tag, int VB, bool STATIC, int UNROLL>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_pack_kernel(const uint8_t *__restrict__ x, size_t n_blocks, int lg_l,
                      const float *__restrict__ block_amax, const float *__restrict__ global_amax,
                      float fp8_max_norm, float six_m, uint2 *__restrict__ packed,
                      uint8_t *__restrict__ scales, float *__restrict__ wsf2_out) {
  // n_blocks counts 16-element chunks; a quant block is 2^lg_l adjacent chunks held by adjacent lanes
  // (block size 16 / 32 / 64 / 128: NVFP4QTensor.quantize takes any block_size, nvfp4_tensor.py:253-342)
  pdl_launch_dependents();
  pdl_wait();
  // weights_scaling_factor_2 = global_amax / (6 * fp8_max)  (nvfp4_tensor.py:104-110, 206-207)
  const float g = global_amax[0];
  // six_m <= 0: the caller hands weights_scaling_factor_2 itself (NVFP4QTensor.quantize(weights_scaling_factor_2=...),
  // nvfp4_tensor.py:262, 281-282) -- used as is, no division
  const float s2 = six_m > 0.f ? __fdiv_rn(g, six_m) : g;
  if (wsf2_out != nullptr && blockIdx.x == 0 && threadIdx.x == 0) wsf2_out[0] = s2;
  const float six_s2 = __fmul_rn(6.0f, s2);
  const ExactDiv d6(six_s2);                                // reciprocal hoisted: 3 FP ops per block instead of a divide
  const float psm = __fdiv_rn(g, 6.0f);
  const size_t base = (size_t)blockIdx.x * (kNvThreads * UNROLL) + threadIdx.x;
  Block<Tag, VB> b[UNROLL];
  float am[UNROLL];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * kNvThreads;
    am[u] = 0.f;
    if (i < n_blocks) {
      b[u].load(x, i);
      if constexpr (STATIC) am[u] = block_amax[i >> lg_l];
    }
  }
#pragma unroll
  for (int u = 0; u < UNROLL; ++u) {
    const size_t i = base + (size_t)u * kNvThreads;
    uint32_t mb = (i < n_blocks) ? Elem<Tag>::absbits_to_f32bits(b[u].absmax_native_bits()) : 0u;
    if (lg_l > 0)
      for (int o = 1; o < (1 << lg_l); o <<= 1) mb = max(mb, __shfl_xor_sync(0xffffffffu, mb, o));
    if (i >= n_blocks) continue;
    float pbs;
    if constexpr (STATIC) {
      // nvfp4_tensor.py:139-161 + _cast_per_block_scale_to_fp8 (:32-48)
      pbs = __fdiv_rn(am[u], 6.0f);
      if (pbs == 0.0f) pbs = 1.0f;
      pbs = __fdiv_rn(__fmul_rn(pbs, fp8_max_norm), psm);
    } else {
      // get_weights_scaling_factor (:169-202)
      pbs = d6.div(__uint_as_float(mb));                   // == __fdiv_rn(amax_b, six_s2)
      if (pbs == 0.0f) pbs = 1.0f;
    }
    // clamp(min=2^-9, max=448) with torch.clamp NaN propagation, then e4m3fn cast
    if (pbs == pbs) pbs = fminf(fmaxf(pbs, 0.001953125f), 448.0f);
    const uint8_t bs8 = f32_to_e4m3fn_torch(pbs);
    if ((i & ((1u << lg_l) - 1u)) == 0) scales[i >> lg_l] = bs8;
    const float denom = __fmul_rn(e4m3_bits_to_f32(bs8), s2);
    packed[i] = encode_block<Tag, VB>(b[u], denom, __uint_as_float(mb));
  }
}

template <typename Tag>
static int launch_nvfp4_pack(const void *x, size_t n_rows, size_t row_len, int block_size, const float *block_amax,
                             const float *global_amax, float fp8_max_norm, bool is_static,
                             uint8_t *packed, uint8_t *scales, float *wsf2_out, cudaStream_t st) {
  const size_t n = n_rows * row_len;
  if (n == 0) return B200Q_OK;
  int lg_l = 0;
  while ((kBlk << lg_l) < block_size) ++lg_l;
  B200Q_REQUIRE((kBlk << lg_l) == block_size && lg_l <= 5, "block_size must be 16, 32, 64, ... 512");
  B200Q_REQUIRE(row_len % (size_t)block_size == 0, "row_len must be a multiple of block_size (pad first, nvfp4_tensor.py:278)");
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x);
  B200Q_REQUIRE(ax % 16 == 0, "x must be 16-byte aligned");
  B200Q_REQUIRE(reinterpret_cast<uintptr_t>(packed) % 8 == 0, "packed must be 8-byte aligned");
  const size_t n_blocks = n / kBlk;
  const int unroll = tuning("pack_unroll", 2) >= 2 ? 2 : 1;
  const size_t per_cta = (size_t)kNvThreads * unroll;
  const size_t grid = (n_blocks + per_cta - 1) / per_cta;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  const float six_m = fp8_max_norm > 0.f ? (float)(6.0 * (double)fp8_max_norm) : 0.f;
  const uint8_t *xb = static_cast<const uint8_t *>(x);
  uint2 *pk = reinterpret_cast<uint2 *>(packed);
  const bool v32 = ax % 32 == 0;
#define LAUNCH(VB_, S_, U_)                                                                        \
  launch_pdl(nvfp4_pack_kernel<Tag, VB_, S_, U_>, dim3((unsigned)grid), dim3(kNvThreads), 0, st, xb, n_blocks, lg_l, block_amax, global_amax, fp8_max_norm, six_m, pk, scales, wsf2_out)
#define LAUNCH_U(VB_, S_)                                                                          \
  do {                                                                                             \
    if (unroll == 2) LAUNCH(VB_, S_, 2);                                                           \
    else LAUNCH(VB_, S_, 1);                                                                       \
  } while (0)
  if (is_static) {
    if (v32) LAUNCH_U(32, true);
    else LAUNCH_U(16, true);
  } else {
    if (v32) LAUNCH_U(32, false);
    else LAUNCH_U(16, false);
  }
#undef LAUNCH_U
#undef LAUNCH
  return check_launch("nvfp4_pack_kernel");
}

// ---------------------------------------------------------------------------------------------
// unpack / dequantize (nvfp4_tensor.py:344-407)
// ---------------------------------------------------------------------------------------------
template <typename Tag>
__global__ void __launch_bounds__(kNvThreads)
    nvfp4_unpack_kernel(const uint2 *__restrict__ packed, const uint8_t *__restrict__ scales,
                        const float *__restrict__ wsf2, uint8_t *__restrict__ y, size_t n_blocks, int lg_l) {
  const size_t i = (size_t)blockIdx.x * kNvThreads + threadIdx.x;
  if (i >= n_blocks) return;
  uint2 c = packed[i];
  {  // the reference LUT maps code 8 (-0) to +0.0 (nvfp4_tensor.py:27): clear the sign of zero codes
    const uint32_t tx = c.x & 0x77777777u, ty = c.y & 0x77777777u;
    c.x = tx | (c.x & ((tx + 0x77777777u) & 0x88888888u));
    c.y = ty | (c.y & ((ty + 0x77777777u) & 0x88888888u));
  }
  const float s = __fmul_rn(e4m3_bits_to_f32(scales[i >> lg_l]), wsf2[0]);
  float f[kBlk];
#pragma unroll
  for (int e = 0; e < kBlk; e += 2) {
    const uint32_t byte = ((e < 8 ? c.x : c.y) >> (4 * (e & 7))) & 0xffu;
    const uint32_t h2 = e2m1x2_to_f16x2(byte);
    f[e] = __fmul_rn(h2f_bits((uint16_t)(h2 & 0xffffu)), s);
    f[e + 1] = __fmul_rn(h2f_bits((uint16_t)(h2 >> 16)), s);
  }
  constexpr int VB = 16;
  constexpr int EPV = VB / Elem<Tag>::SIZE;
  Vec<VB> *out = reinterpret_cast<Vec<VB> *>(y) + i * (kBlk / EPV);
#pragma unroll
  for (int k = 0; k < kBlk / EPV; ++k) {
    Vec<VB> v;
    floats_to_vec<Tag, VB>(f + k * EPV, v);
    stg(out + k, v);
  }
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_fake_quant_nvfp4(const void *x, void *y, int dtype, size_t n_rows, size_t row_len,
                           const void *global_amax, int amax_dtype, b200q_stream_t stream) {
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n_rows * row_len == 0, "null tensor");
  B200Q_REQUIRE(global_amax != nullptr && dtype_ok(amax_dtype), "global_amax is null or has a bad dtype");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_dyn<Tag>(x, y, n_rows, row_len, global_amax, amax_dtype,
                                                    (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_fake_quant_nvfp4_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, const void *amax_base,
                                 int amax_dtype, b200q_stream_t stream) {
  if (n_desc == 0 || total_ctas == 0) return B200Q_OK;
  B200Q_REQUIRE(descs != nullptr && amax_base != nullptr && n_desc > 0, "null pointer");
  B200Q_REQUIRE(total_ctas <= 0x7fffffffu, "too many CTAs");
  const MultiDesc *d = static_cast<const MultiDesc *>(descs);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       launch_pdl(nvfp4_dyn_multi_kernel<Tag, 32, 2, false>, dim3((unsigned)total_ctas), dim3(kNvThreads),
                                  0, (cudaStream_t)stream, d, n_desc, amax_base, amax_dtype, nullptr));
  return check_launch("nvfp4_dyn_multi_kernel");
}

int b200q_collect_fake_quant_nvfp4_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, float *slots,
                                         const void *amax_base, int amax_dtype, b200q_stream_t stream) {
  if (n_desc == 0 || total_ctas == 0) return B200Q_OK;
  B200Q_REQUIRE(descs != nullptr && slots != nullptr && amax_base != nullptr && n_desc > 0, "null pointer");
  B200Q_REQUIRE(dtype_ok(amax_dtype), "unknown amax dtype %d", amax_dtype);
  B200Q_REQUIRE(total_ctas <= 0x7fffffffu, "too many CTAs");
  const MultiDesc *d = static_cast<const MultiDesc *>(descs);
  uint32_t *sl = reinterpret_cast<uint32_t *>(slots);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       launch_pdl(nvfp4_dyn_multi_kernel<Tag, 32, 2, true>, dim3((unsigned)total_ctas), dim3(kNvThreads),
                                  0, (cudaStream_t)stream, d, n_desc, amax_base, amax_dtype, sl));
  return check_launch("nvfp4_dyn_multi_kernel<collect>");
}

int b200q_fake_quant_nvfp4_multi_fixup(const void *descs, const void *live, int n_desc, int dtype,
                                       const float *slots, const void *amax_base, int amax_dtype, const void *pieces,
                                       int n_pieces, int *redo_count, b200q_stream_t stream) {
  if (n_desc == 0) return B200Q_OK;
  B200Q_REQUIRE(descs != nullptr && live != nullptr && slots != nullptr && amax_base != nullptr &&
                    (pieces != nullptr || n_pieces == 0) && redo_count != nullptr && n_desc > 0 && n_pieces >= 0,
                "null pointer");
  B200Q_REQUIRE(dtype_ok(amax_dtype), "unknown amax dtype %d", amax_dtype);
  const MultiDesc *d = static_cast<const MultiDesc *>(descs);
  const unsigned long long *lf = static_cast<const unsigned long long *>(live);
  const uint32_t *sl = reinterpret_cast<const uint32_t *>(slots);
  const long long *pc = static_cast<const long long *>(pieces);
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_fixup<Tag>(d, lf, n_desc, sl, amax_base, amax_dtype, pc, n_pieces, redo_count,
                                                      (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_fake_quant_nvfp4_static(const void *x, void *y, int dtype, size_t n_blocks,
                                  int block_size, const float *block_amax,
                                  const float *global_amax, int quantize_block_scales,
                                  float fp8_max_norm, b200q_stream_t stream) {
  B200Q_REQUIRE((x != nullptr && y != nullptr) || n_blocks == 0, "null tensor");
  B200Q_REQUIRE(block_size == kBlk, "only block_size 16 is supported (got %d)", block_size);
  B200Q_REQUIRE(block_amax != nullptr, "block_amax is null");
  B200Q_REQUIRE(!quantize_block_scales || global_amax != nullptr, "global_amax is required to quantize block scales");
  B200Q_REQUIRE(fp8_max_norm > 0.f, "fp8_max_norm must be positive");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_static<Tag>(x, y, n_blocks, block_amax, global_amax,
                                                       quantize_block_scales, fp8_max_norm,
                                                       (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_pack_nvfp4(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                     const float *global_amax, uint8_t *packed, uint8_t *scales_e4m3,
                     float *wsf2_out, b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n_rows * row_len == 0, "x is null");
  B200Q_REQUIRE(global_amax != nullptr && packed != nullptr && scales_e4m3 != nullptr, "null pointer");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_pack<Tag>(x, n_rows, row_len, block_size, nullptr, global_amax, 448.0f,
                                                     false, packed, scales_e4m3, wsf2_out,
                                                     (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_pack_nvfp4_scale2(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                            const float *wsf2, uint8_t *packed, uint8_t *scales_e4m3, b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n_rows * row_len == 0, "x is null");
  B200Q_REQUIRE(wsf2 != nullptr && packed != nullptr && scales_e4m3 != nullptr, "null pointer");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_pack<Tag>(x, n_rows, row_len, block_size, nullptr, wsf2, 0.0f,
                                                     false, packed, scales_e4m3, nullptr,
                                                     (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_pack_nvfp4_static(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                            const float *block_amax, const float *global_amax,
                            float fp8_max_norm, uint8_t *packed, uint8_t *scales_e4m3,
                            float *wsf2_out, b200q_stream_t stream) {
  B200Q_REQUIRE(x != nullptr || n_rows * row_len == 0, "x is null");
  B200Q_REQUIRE(block_amax != nullptr && global_amax != nullptr && packed != nullptr && scales_e4m3 != nullptr, "null pointer");
  B200Q_REQUIRE(fp8_max_norm > 0.f, "fp8_max_norm must be positive");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       return launch_nvfp4_pack<Tag>(x, n_rows, row_len, block_size, block_amax, global_amax,
                                                     fp8_max_norm, true, packed, scales_e4m3,
                                                     wsf2_out, (cudaStream_t)stream));
  return B200Q_OK;
}

int b200q_unpack_nvfp4(const uint8_t *packed, const uint8_t *scales_e4m3, const float *wsf2,
                       void *y, int dtype, size_t n_rows, size_t row_len, int block_size, b200q_stream_t stream) {
  const size_t n = n_rows * row_len;
  if (n == 0) return B200Q_OK;
  B200Q_REQUIRE(packed != nullptr && scales_e4m3 != nullptr && wsf2 != nullptr && y != nullptr, "null pointer");
  int lg_l = 0;
  while ((kBlk << lg_l) < block_size) ++lg_l;
  B200Q_REQUIRE((kBlk << lg_l) == block_size && lg_l <= 5, "block_size must be 16, 32, 64, ... 512");
  B200Q_REQUIRE(row_len % (size_t)block_size == 0, "row_len must be a multiple of block_size");
  B200Q_REQUIRE(reinterpret_cast<uintptr_t>(packed) % 8 == 0 && reinterpret_cast<uintptr_t>(y) % 16 == 0, "packed / y alignment");
  const size_t n_blocks = n / kBlk;
  const size_t grid = (n_blocks + kNvThreads - 1) / kNvThreads;
  B200Q_REQUIRE(grid <= 0x7fffffffu, "tensor too large");
  B200Q_DISPATCH_DTYPE(dtype, Tag,
                       nvfp4_unpack_kernel<Tag><<<(unsigned)grid, kNvThreads, 0, (cudaStream_t)stream>>>(
                           reinterpret_cast<const uint2 *>(packed), scales_e4m3, wsf2,
                           static_cast<uint8_t *>(y), n_blocks, lg_l));
  return check_launch("nvfp4_unpack_kernel");
}

}  // extern "C"
