// hist_search.cu -- amax search over a collected histogram on the GPU (SURVEY.md 8(f2)).
//
// Reference: HistogramCalibrator.compute_amax -> _compute_amax_entropy / _mse / _percentile
// (quantization/calib/histogram.py:137-343): host-side NumPy / Python, the entropy search an O(bins^2) Python
// loop (seconds per quantizer at 2048 bins).  Here every candidate threshold is one CTA.
//
//   percentile  cdf = cumsum(hist / total) sequentially in fp64 (np.cumsum adds left to right), left searchsorted
//   entropy     for i in range(start_bin, nbins + 1, stride): KL(reference_density || quantized density), fp64;
//               bucket membership = np.digitize(range(i), np.linspace(0, i, nq + 1)) - 1 restated exactly
//               (linspace entries are k * fl(i / nq) in fp64, the last one i); bucket sums are integer counts,
//               exact in int64 prefix sums; the remaining fp64 sums are accumulated in a different order than
//               NumPy's pairwise summation (1e-15 relative)
//   mse         for i in range(start_bin, n_centers, stride): mean((fq(c; amax = c_i) - c)^2 * counts) in fp32
//               element arithmetic like torch, fp64 accumulation; fq = the integer / FP8 fake quant of
//               kernels/quantization/gemm/tensor_quant_gpu.cu:38-73 / tensor_quant_gpu_fp8.cu:90-107 with the default
//               narrow_range=True (the reference's call site, with its positional-argument slip repaired: see
//               DESIGN.md section 4)
#include "intq.cuh"

namespace b200q {

constexpr int kHsThreads = 256;

__device__ __forceinline__ double block_sum_f64(double v, double *s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kHsThreads / 32; ++w) t += s_red[w];      // same order in every thread
  return t;
}

// ---- percentile ---------------------------------------------------------------------------------
__global__ void hist_percentile_kernel(const float *__restrict__ hist, int nbins, double target, int *__restrict__ idx_out) {
  long long total = 0;
  for (int i = 0; i < nbins; ++i) total += (long long)hist[i];
  double cdf = 0.0;
  int idx = nbins;
  for (int i = 0; i < nbins; ++i) {
    cdf += (double)(long long)hist[i] / (double)total;
    if (cdf >= target) {
      idx = i;
      break;
    }
  }
  idx_out[0] = idx;
}

// ---- entropy --------------------------------------------------------------------------------------
// prefix[0..nbins]: int64 counts with bins[0] = bins[1] (histogram.py:221-222); nzc[0..nbins]: non-zero bins before
__global__ void hist_prefix_kernel(const float *__restrict__ hist, int nbins, long long *__restrict__ prefix,
                                   int *__restrict__ nzc) {
  long long p = 0;
  int c = 0;
  prefix[0] = 0;
  nzc[0] = 0;
  for (int i = 0; i < nbins; ++i) {
    const long long b = (long long)hist[(i == 0 && nbins > 1) ? 1 : i];
    p += b;
    c += b != 0;
    prefix[i + 1] = p;
    nzc[i + 1] = c;
  }
}

__global__ void __launch_bounds__(kHsThreads)
    hist_entropy_kernel(const long long *__restrict__ prefix, const int *__restrict__ nzc, int nbins, int nq,
                        int start_bin, int stride, double *__restrict__ div_out) {
  __shared__ double s_red[kHsThreads / 32];
  const int i = start_bin + (int)blockIdx.x * stride;            // candidate threshold: bins [0, i) are kept
  const double di = (double)i;
  const double step = di / (double)nq;                            // np.linspace(0, i, nq + 1): step = i / nq
  auto space = [&](int k) { return k >= nq ? di : (double)k * step; };
  auto bin_at = [&](int idx) { return prefix[idx + 1] - prefix[idx]; };
  auto density = [&](int idx) -> double {                         // new_density[idx] (:245-261)
    if (bin_at(idx) == 0) return 0.0;
    int k = (int)((double)idx / step);
    if (k > nq - 1) k = nq - 1;
    while (k + 1 <= nq - 1 && space(k + 1) <= (double)idx) ++k;   // digitize: space(k) <= idx < space(k + 1)
    while (k > 0 && space(k) > (double)idx) --k;
    const int lo = (int)ceil(space(k));
    const int hi = (k + 1 >= nq) ? i : (int)ceil(space(k + 1));
    return (double)(prefix[hi] - prefix[lo]) / (double)(nzc[hi] - nzc[lo]);
  };
  double sq = 0.0;
  for (int idx = threadIdx.x; idx < i; idx += kHsThreads) sq += density(idx);
  const double sum_q = block_sum_f64(sq, s_red);
  const long long tail = prefix[nbins] - prefix[i];
  const double total = (double)prefix[nbins];                     // == sum(reference_density)
  double kl = 0.0;
  for (int idx = threadIdx.x; idx < i; idx += kHsThreads) {
    const long long r = bin_at(idx) + (idx == i - 1 ? tail : 0);
    if (r > 0) {                                                  // rel_entr(p, q) = p * log(p / q), 0 where p == 0
      const double p = (double)r / total;
      const double q = density(idx) / sum_q;
      kl += p * log(p / q);
    }
  }
  kl = block_sum_f64(kl, s_red);
  if (threadIdx.x == 0) div_out[blockIdx.x] = kl;
}

// ---- mse ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kHsThreads)
    hist_mse_kernel(const float *__restrict__ hist, const float *__restrict__ centers, int n, int num_bits,
                    float max_bound, float min_bound, int start_bin, int stride, float *__restrict__ mse_out) {
  __shared__ double s_red[kHsThreads / 32];
  const int i = start_bin + (int)blockIdx.x * stride;
  const float amax = centers[i];
  IntQ q;
  Fp8Scale fs;
  if (num_bits > 0) q.setup(amax, max_bound, min_bound);
  else fs.setup(amax);
  double acc = 0.0;
  for (int idx = threadIdx.x; idx < n; idx += kHsThreads) {
    const float c = centers[idx];
    const float qc = num_bits > 0 ? q.apply(c) : fs.apply(c);
    const float d = __fsub_rn(qc, c);
    acc += (double)__fmul_rn(__fmul_rn(d, d), (float)(long long)hist[idx]);
  }
  acc = block_sum_f64(acc, s_red);
  if (threadIdx.x == 0) mse_out[blockIdx.x] = (float)(acc / (double)n);
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_hist_search_percentile(const float *hist, int nbins, double percentile, int *idx_out, b200q_stream_t stream) {
  B200Q_REQUIRE(hist != nullptr && idx_out != nullptr && nbins > 0, "bad arguments");
  B200Q_REQUIRE(percentile >= 0.0 && percentile <= 100.0, "Invalid percentile. Must be in range 0 <= percentile <= 100.");
  hist_percentile_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(hist, nbins, percentile / 100.0, idx_out);
  return check_launch("hist_percentile_kernel");
}

int b200q_hist_search_entropy(const float *hist, int nbins, int num_quant_bins, int stride, int start_bin,
                              long long *prefix_scratch, int *nz_scratch, double *div_out, b200q_stream_t stream) {
  B200Q_REQUIRE(hist != nullptr && prefix_scratch != nullptr && nz_scratch != nullptr && div_out != nullptr, "null pointer");
  B200Q_REQUIRE(nbins > 1 && num_quant_bins > 0 && stride > 0 && start_bin > 0 && start_bin <= nbins, "bad arguments");
  const int n_cand = (nbins - start_bin) / stride + 1;           // range(start_bin, nbins + 1, stride)
  cudaStream_t st = (cudaStream_t)stream;
  hist_prefix_kernel<<<1, 1, 0, st>>>(hist, nbins, prefix_scratch, nz_scratch);
  hist_entropy_kernel<<<n_cand, kHsThreads, 0, st>>>(prefix_scratch, nz_scratch, nbins, num_quant_bins, start_bin, stride, div_out);
  return check_launch("hist_entropy_kernel");
}

int b200q_hist_search_mse(const float *hist, const float *centers, int n_centers, int num_bits, int is_unsigned,
                          int stride, int start_bin, float *mse_out, b200q_stream_t stream) {
  B200Q_REQUIRE(hist != nullptr && centers != nullptr && mse_out != nullptr, "null pointer");
  B200Q_REQUIRE(n_centers > 0 && stride > 0 && start_bin >= 0 && start_bin < n_centers, "bad arguments");
  B200Q_REQUIRE(num_bits >= 0 && num_bits <= 16, "unsupported num_bits %d", num_bits);
  float maxb = 0.f, minb = 0.f;
  if (num_bits > 0) {
    maxb = (float)((1 << (num_bits - 1 + (is_unsigned ? 1 : 0))) - 1);
    minb = -maxb;                                                // narrow_range=True, the function's default
  }
  const int n_cand = (n_centers - 1 - start_bin) / stride + 1;   // range(start_bin, n_centers, stride)
  hist_mse_kernel<<<n_cand, kHsThreads, 0, (cudaStream_t)stream>>>(hist, centers, n_centers, num_bits, maxb, minb,
                                                                  start_bin, stride, mse_out);
  return check_launch("hist_mse_kernel");
}

}  // extern "C"
