// runtime.cu -- library plumbing: error strings, device info, tuning knobs, self tests.
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"

namespace b200q {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char *what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return B200Q_ERR_CUDA;
  }
  return B200Q_OK;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

struct Knob {
  const char *key;
  int value;
};
static Knob g_knobs[] = {
    {"amax_unroll", 0}, {"ew_unroll", 0}, {"vec_bytes", 0}, {"amax_ctas_per_sm", 0},
    {"nvfp4_unroll", 0}, {"hist_ctas_per_sm", 0}, {"pdl", 0}, {"pack_unroll", 0}, {"amax_tma", 0}, {"tma_tile_kb", 0}, {"tma_stages", 0}, {"tma_ctas_per_sm", 0}, {"nvfp4_tma_store", 0}, {"hist_variant", 0}, {"nf4_lut", 0}, {"hist_hot", 0},
};

int tuning(const char *key, int dflt) {
  for (auto &k : g_knobs)
    if (strcmp(k.key, key) == 0) return k.value != 0 ? k.value : dflt;
  return dflt;
}

// ---- fastdiv self test ---------------------------------------------------------------------
__device__ __forceinline__ uint64_t splitmix(uint64_t &s) {
  uint64_t z = (s += 0x9e3779b97f4a7c15ull);
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__global__ void fastdiv_selftest_kernel(uint64_t seed, size_t n, unsigned long long *mism) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t s = seed + i * 0x632be59bd9b4e019ull;
  const uint64_t r0 = splitmix(s), r1 = splitmix(s);
  // divisor: random positive float with exponent in a wide window; every 4th one gets an
  // all-ones / all-zeros / sparse mantissa (the classic hard cases for reciprocal methods)
  uint32_t bm = (uint32_t)(r0 & 0x7fffffu);
  const uint32_t kind = (uint32_t)(r0 >> 60);
  if (kind == 0) bm = 0x7fffffu;
  if (kind == 1) bm = 0;
  if (kind == 2) bm &= 0x700000u;
  if (kind == 3) bm |= 0x7ffff0u;
  const int be = 127 - 70 + (int)((r0 >> 24) % 140);  // 2^-70 .. 2^69
  const float b = __uint_as_float(((uint32_t)be << 23) | bm);
  // dividend: bf16-like (8 significant bits) half the time, full fp32 otherwise; near b * {E2M1
  // midpoints} a quarter of the time so exact ties are exercised
  uint32_t am = (uint32_t)(r1 & 0x7fffffu);
  if (r1 >> 63) am &= 0x7f0000u;
  int ae = be - 4 + (int)((r1 >> 24) % 9);
  if (ae < 1) ae = 1;
  if (ae > 254) ae = 254;
  float a = __uint_as_float(((uint32_t)ae << 23) | am);
  const uint32_t k2 = (uint32_t)((r1 >> 40) & 15u);
  const float mids[8] = {0.25f, 0.75f, 1.25f, 1.75f, 2.5f, 3.5f, 5.0f, 127.5f};
  if (k2 < 4) a = b * mids[(r1 >> 44) & 7u];
  if ((r1 >> 50) & 1u) a = -a;
  ExactDiv d(b);
  const float q1 = d.div(a);
  const float q2 = __fdiv_rn(a, b);
  if (__float_as_uint(q1) != __float_as_uint(q2)) atomicAdd(mism, 1ull);
}

// ---- E2M1 rounding self test ---------------------------------------------------------------
// one thread per non-negative fp32 bit pattern (every finite value, +inf and the NaNs): the branch-free
// e2m1_round_mag against the reference's compare chain, bit for bit
__global__ void e2m1_round_selftest_kernel(unsigned long long *mism) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  const float a = __uint_as_float(u);
  if (__float_as_uint(e2m1_round_mag(a)) != __float_as_uint(e2m1_round_mag_ref(a))) atomicAdd(mism, 1ull);
}

}  // namespace b200q

using namespace b200q;

extern "C" {

int b200q_version(void) { return B200Q_VERSION; }

const char *b200q_last_error(void) { return g_err; }

int b200q_device_info(int *sm_count_out, int *cc_major, int *cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error("cudaGetDevice: %s", cudaGetErrorString(e));
    return B200Q_ERR_CUDA;
  }
  int n = 0, ma = 0, mi = 0;
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&ma, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&mi, cudaDevAttrComputeCapabilityMinor, dev);
  if (sm_count_out) *sm_count_out = n;
  if (cc_major) *cc_major = ma;
  if (cc_minor) *cc_minor = mi;
  return B200Q_OK;
}

int b200q_set_device(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    set_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    return B200Q_ERR_CUDA;
  }
  return B200Q_OK;
}

int b200q_set_tuning(const char *key, int value) {
  if (!key) return B200Q_ERR_INVALID;
  for (auto &k : g_knobs)
    if (strcmp(k.key, key) == 0) {
      k.value = value;
      return B200Q_OK;
    }
  set_error("unknown tuning key '%s'", key);
  return B200Q_ERR_INVALID;
}

int b200q_get_tuning(const char *key, int *value) {
  if (!key || !value) return B200Q_ERR_INVALID;
  for (auto &k : g_knobs)
    if (strcmp(k.key, key) == 0) {
      *value = k.value;
      return B200Q_OK;
    }
  set_error("unknown tuning key '%s'", key);
  return B200Q_ERR_INVALID;
}

int b200q_selftest_fastdiv(uint64_t seed, size_t n, unsigned long long *mismatches_host) {
  B200Q_REQUIRE(mismatches_host != nullptr, "mismatches_host is null");
  unsigned long long *d = nullptr;
  if (cudaMalloc(&d, sizeof(*d)) != cudaSuccess) {
    set_error("cudaMalloc failed");
    return B200Q_ERR_CUDA;
  }
  cudaMemset(d, 0, sizeof(*d));
  const int threads = 256;
  const size_t blocks = (n + threads - 1) / threads;
  if (blocks > 0) fastdiv_selftest_kernel<<<(unsigned)blocks, threads>>>(seed, n, d);
  int rc = check_launch("fastdiv_selftest");
  cudaMemcpy(mismatches_host, d, sizeof(*d), cudaMemcpyDeviceToHost);
  cudaFree(d);
  return rc;
}

int b200q_selftest_e2m1_round(unsigned long long *mismatches_host) {
  B200Q_REQUIRE(mismatches_host != nullptr, "mismatches_host is null");
  unsigned long long *d = nullptr;
  if (cudaMalloc(&d, sizeof(*d)) != cudaSuccess) {
    set_error("cudaMalloc failed");
    return B200Q_ERR_CUDA;
  }
  cudaMemset(d, 0, sizeof(*d));
  const int threads = 256;
  e2m1_round_selftest_kernel<<<(1u << 31) / threads, threads>>>(d);  // 2^31 patterns: sign bit clear
  int rc = check_launch("e2m1_round_selftest");
  cudaMemcpy(mismatches_host, d, sizeof(*d), cudaMemcpyDeviceToHost);
  cudaFree(d);
  return rc;
}

}  // extern "C"
