// gptq.cu -- the column loop of one GPTQ block in one kernel.
//
// Reference semantics: gptq_blockwise_update (quantization/utils/calib_utils.py:241-276), the unfused loop the
// reference's GPTQHelper runs.  For a block [bs, be) with U = Hinv[bs:be, bs:be] and i = 0 .. nb-1 in order:
//   q = Q(w[:, bs+i]);  W[:, bs+i] = q;  err = (w_i - q) / U[i,i];  w_j -= err * U[i,j] for j >= i;  E[:, i] = err
// where Q is the weight quantizer's fake quant of the fp32 working matrix.  The update is the arithmetic of ATen's
// CUDA addr_ kernel as ptxas compiled it (LinearAlgebra.cu, addr_kernel_cuda: FMUL alpha*vec1, FMUL *vec2, FFMA
// self*beta + product): the product err * U[i,j] is rounded, then added -- NOT one fused multiply-add.  The trailing
// update W[:, be:] -= E @ Hinv[bs:be, be:] stays a cuBLAS GEMM on the host side.
//
// Every output row is independent: the in-block recurrence only touches its own row, and for every covered format the
// scale of an element depends on calibrated state or on the element's own row (NVFP4 dynamic: its 16-element block).
// Layout: one warp per row, lane l holds columns 4l .. 4l+3 of the block in registers (nb <= 128), so a 16-element
// NVFP4 block is 4 lanes and its amax two shuffles.  Per column the owning lane quantizes, divides and broadcasts the
// error; every lane then updates its own columns from U, which is staged in shared memory once per CTA (upper
// triangle only, zeros below).  Each CTA loops its 8 warps over row tiles.
#include "block16.cuh"
#include "intq.cuh"

namespace b200q {

constexpr int kGptqThreads = 256;   // 8 warps: 8 rows in flight per CTA
constexpr int kGptqMaxCols = 128;   // 32 lanes x 4 columns

enum : int { kGptqInt = 0, kGptqFp8 = 1, kGptqNvfp4Static = 2, kGptqNvfp4Dyn = 3 };

struct GptqArgs {
  float *w;                 // [rows, ldw], the block's first column at w[0]
  size_t ldw, rows;
  int nb;
  const float *u;           // [nb, ldu], upper triangle read
  size_t ldu;
  float *e;                 // [rows, nb]
  const void *amax;         // INT / FP8: amax[row * amax_row_stride + (col0 + c) / amax_col_block]
  int amax_dtype;           // NVFP4 static: fp32 block amax, same indexing; NVFP4 dynamic: the per-tensor amax
  size_t amax_row_stride, amax_col_block, col0;
  float max_bound, min_bound;
  const float *global_amax; // NVFP4 static
};

template <int FMT>
__global__ void __launch_bounds__(kGptqThreads) gptq_block_kernel(GptqArgs a) {
  extern __shared__ __align__(16) float s_u[];
  const int nb = a.nb;
  const int sp = (nb + 3) & ~3;  // row pitch of the staged U: float4 reads at 4 * lane
  for (int idx = threadIdx.x; idx < nb * sp; idx += kGptqThreads) {
    const int i = idx / sp, j = idx - i * sp;
    s_u[idx] = (j >= i && j < nb) ? a.u[(size_t)i * a.ldu + j] : 0.f;
  }
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int c_lo = lane * 4;
  const bool has_cols = c_lo < nb;
  const size_t n_warps = (size_t)gridDim.x * (kGptqThreads / 32);

  StaticScale ss;
  ss.setup(a.global_amax, FMT == kGptqNvfp4Static, 1.0f);
  DynScale ds;
  ds.setup(FMT == kGptqNvfp4Dyn ? load_scalar(a.amax, a.amax_dtype, 0) : 1.0f);
  const ExactDiv d6(ds.six_gs);

  for (size_t r = (size_t)blockIdx.x * (kGptqThreads / 32) + (threadIdx.x >> 5); r < a.rows; r += n_warps) {
    float *wr = a.w + r * a.ldw;
    float w[4], qv[4], ev[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      w[k] = (c_lo + k < nb) ? wr[c_lo + k] : 0.f;
      qv[k] = ev[k] = 0.f;
    }
    // scales that do not depend on the working values, set up once per row
    IntQ iq[4];
    Fp8Scale fs[4];
    if constexpr (FMT == kGptqInt || FMT == kGptqFp8) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const size_t c = a.col0 + c_lo + k;
        const float am =
            (c_lo + k < nb) ? load_scalar(a.amax, a.amax_dtype, r * a.amax_row_stride + c / a.amax_col_block) : 1.f;
        if constexpr (FMT == kGptqInt) iq[k].setup(am, a.max_bound, a.min_bound);
        else fs[k].setup(am);
      }
    }
    float s_st = 1.f;
    bool zero_st = false;
    if constexpr (FMT == kGptqNvfp4Static) {  // the lane's 4 columns lie in one 16-element block
      const float s = has_cols ? ss.block_scale(((const float *)a.amax)[r * a.amax_row_stride + (a.col0 + c_lo) / kBlk])
                               : 1.f;
      s_st = static_block_scale_safe(s, zero_st);
    }
    const ExactDiv dst(s_st);

    for (int i0 = 0; i0 < nb; i0 += 4) {
      const int owner = i0 >> 2;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = i0 + k;
        if (i >= nb) break;  // warp-uniform
        uint32_t mb = 0;     // |w| max of the 16-element block, as fp32 bits (NaN-propagating)
        uint32_t mn = 0;     // 1 + the bits of the NaN-ignoring |w| max (dyn_block_max); 0: every element is NaN
        if constexpr (FMT == kGptqNvfp4Static || FMT == kGptqNvfp4Dyn) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t a = __float_as_uint(w[kk]) & 0x7fffffffu;
            mb = max(mb, a);
            mn = max(mn, a <= 0x7f800000u ? a + 1u : 0u);
          }
          mb = group_max<4>(mb);
          if constexpr (FMT == kGptqNvfp4Dyn) mn = group_max<4>(mn);
        }
        float err = 0.f;
        if (lane == owner) {
          const float x = w[k];
          float q;
          if constexpr (FMT == kGptqInt) {
            q = iq[k].apply(x);
          } else if constexpr (FMT == kGptqFp8) {
            q = fs[k].apply(x);
          } else if constexpr (FMT == kGptqNvfp4Static) {
            q = zero_st ? 0.f : qdq_e2m1_one(__fadd_rn(x, 0.f), dst, dst.block_ok(mb < 0x7f800000u));
          } else {
            const ExactDiv d(ds.block_scale(mn ? __uint_as_float(mn - 1u) : __uint_as_float(0x7fc00000u), d6));
            q = qdq_e2m1_one(__fadd_rn(x, 0.f), d, d.block_ok(mb < 0x7f800000u));
          }
          err = __fdiv_rn(__fsub_rn(x, q), s_u[i * sp + i]);
          qv[k] = q;
          ev[k] = err;
        }
        err = __shfl_sync(0xffffffffu, err, owner);
        if (has_cols) {
          const float4 u4 = *reinterpret_cast<const float4 *>(&s_u[i * sp + c_lo]);
          const float uu[4] = {u4.x, u4.y, u4.z, u4.w};
          const float ne = -err;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            if (c_lo + kk >= i && c_lo + kk < nb) w[kk] = __fadd_rn(w[kk], __fmul_rn(ne, uu[kk]));
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (c_lo + k < nb) {
        wr[c_lo + k] = qv[k];
        a.e[r * (size_t)nb + c_lo + k] = ev[k];
      }
    }
  }
}

template <int FMT> static int launch_gptq(const GptqArgs &a, cudaStream_t st) {
  auto kern = gptq_block_kernel<FMT>;
  const size_t smem = sizeof(float) * (size_t)a.nb * (size_t)((a.nb + 3) & ~3);
  // the opt-in above 48 KB is a property of the function on the CURRENT device: set on every such launch
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("gptq_block_kernel (shared-memory opt-in)");
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kGptqThreads, smem) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  const size_t rows_per_cta = kGptqThreads / 32;
  size_t grid = (a.rows + rows_per_cta - 1) / rows_per_cta;
  const size_t cap = (size_t)sm_count() * (size_t)per_sm;
  if (grid > cap) grid = cap;
  kern<<<(unsigned)grid, kGptqThreads, smem, st>>>(a);
  return check_launch("gptq_block_kernel");
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_gptq_block(float *w, size_t ldw, size_t rows, int nb, const float *u, size_t ldu, float *e, int fmt,
                     const void *amax, int amax_dtype, size_t amax_row_stride, size_t amax_col_block, size_t col0,
                     int num_bits, int is_unsigned, int narrow_range, const float *global_amax,
                     b200q_stream_t stream) {
  B200Q_REQUIRE(nb >= 1 && nb <= kGptqMaxCols, "nb must be in [1, %d], got %d", kGptqMaxCols, nb);
  if (rows == 0) return B200Q_OK;
  B200Q_REQUIRE(w != nullptr && u != nullptr && e != nullptr, "null tensor");
  B200Q_REQUIRE(ldw >= (size_t)nb && ldu >= (size_t)nb, "leading dimensions must be >= nb");
  B200Q_REQUIRE(amax != nullptr && dtype_ok(amax_dtype), "amax is null or has a bad dtype");
  GptqArgs a;
  a.w = w;
  a.ldw = ldw;
  a.rows = rows;
  a.nb = nb;
  a.u = u;
  a.ldu = ldu;
  a.e = e;
  a.amax = amax;
  a.amax_dtype = amax_dtype;
  a.amax_row_stride = amax_row_stride;
  a.amax_col_block = amax_col_block;
  a.col0 = col0;
  a.max_bound = a.min_bound = 0.f;
  a.global_amax = global_amax;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (fmt) {
  case kGptqInt: {
    B200Q_REQUIRE(num_bits >= 1 && num_bits + (is_unsigned ? 1 : 0) <= 24, "unsupported num_bits %d", num_bits);
    B200Q_REQUIRE(amax_col_block >= 1, "amax_col_block must be >= 1");
    // bits_to_bound (tensor_quant_gpu.cu:38-41), as b200q_fake_quant_int
    const float bound = (float)((1 << (num_bits - 1 + (is_unsigned ? 1 : 0))) - 1);
    a.max_bound = bound;
    a.min_bound = -(bound + (narrow_range ? 0.f : 1.f));
    return launch_gptq<kGptqInt>(a, st);
  }
  case kGptqFp8:
    B200Q_REQUIRE(amax_col_block >= 1, "amax_col_block must be >= 1");
    return launch_gptq<kGptqFp8>(a, st);
  case kGptqNvfp4Static:
    B200Q_REQUIRE(amax_dtype == B200Q_F32 && global_amax != nullptr, "static NVFP4 needs fp32 block amax and global_amax");
    B200Q_REQUIRE(amax_col_block == (size_t)kBlk, "static NVFP4 block amax must be per 16 columns");
    B200Q_REQUIRE(nb % kBlk == 0 && col0 % kBlk == 0, "NVFP4 blocks must not straddle the GPTQ block (nb %d, col0 %zu)",
                  nb, col0);
    return launch_gptq<kGptqNvfp4Static>(a, st);
  case kGptqNvfp4Dyn:
    B200Q_REQUIRE(nb % kBlk == 0 && col0 % kBlk == 0, "NVFP4 blocks must not straddle the GPTQ block (nb %d, col0 %zu)",
                  nb, col0);
    return launch_gptq<kGptqNvfp4Dyn>(a, st);
  default:
    B200Q_REQUIRE(false, "unknown GPTQ quantizer format %d", fmt);
  }
  return B200Q_OK;
}

}  // extern "C"
