/*
 * b200quant.h -- C-ABI of the H100-native PTQ calibration / fake-quant / quant-and-pack engine.
 *
 * This header is the drop-in boundary for the hot path named in BASELINE.json: every entry point
 * is what a binding of NVIDIA/Model-Optimizer's quantization extension modules would call.  Each
 * declaration cites the reference interface it replaces (paths relative to the reference tree,
 * modelopt/torch/...).  No torch types cross this boundary: plain device pointers, element
 * counts, a CUDA stream handle, `int` status.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - `dtype` is a b200q_dtype (element type of the tensor being read / written);
 *   - all work is enqueued on `stream` (a cudaStream_t / CUstream); nothing synchronises;
 *   - return value: B200Q_OK or a B200Q_ERR_* code; b200q_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - "amax slots" are fp32 values holding a non-negative running maximum.  Collect kernels do
 *     slot = max(slot, local) with an unsigned-integer atomic on the bit pattern, which is exact
 *     for non-negative floats and orders NaN above +inf, i.e. a NaN anywhere in the input makes
 *     the slot NaN (the reference's torch.max/torch.min propagate NaN the same way,
 *     quantization/utils/core_utils.py:172-174).  Zero a slot to start a new calibration.
 */
#ifndef B200QUANT_H_
#define B200QUANT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200Q_VERSION 100 /* 0.1.0 */

#define B200Q_OK 0
#define B200Q_ERR_INVALID 1     /* bad argument (null pointer, size mismatch, unknown enum) */
#define B200Q_ERR_UNSUPPORTED 2 /* valid request this build has no kernel for */
#define B200Q_ERR_CUDA 3        /* a CUDA runtime call or launch failed */

typedef enum { B200Q_F32 = 0, B200Q_F16 = 1, B200Q_BF16 = 2 } b200q_dtype;

typedef struct CUstream_st *b200q_stream_t; /* == cudaStream_t */

/* ---- library ---------------------------------------------------------------------------- */
int b200q_version(void);
const char *b200q_last_error(void);
/* Device properties of the current device (SM count, compute capability). */
int b200q_device_info(int *sm_count, int *cc_major, int *cc_minor);
/* Make `device` current for this library's CUDA runtime instance (the library links cudart
 * statically; call it when the host framework switches devices). */
int b200q_set_device(int device);
/* Launch-shape tuning knob (bench / autotune only).  key: "amax_unroll", "ew_unroll", "vec_bytes". */
int b200q_set_tuning(const char *key, int value);
/* The value a knob holds (0: unset, the built-in default applies). */
int b200q_get_tuning(const char *key, int *value);

/* ---- (1) calibration collect ------------------------------------------------------------ */

/* Per-tensor |x| maximum, fused with the calibrator's running max:
 *   amax_slot[0] = max(amax_slot[0], max_i |x_i|)
 * Replaces reduce_amax(x, axis=None) (quantization/utils/core_utils.py:147-183) + the
 * torch.max update in MaxCalibrator.collect (quantization/calib/max.py:53-86). */
int b200q_amax_per_tensor(const void *x, int dtype, size_t n, float *amax_slot,
                          b200q_stream_t stream);

/* Segmented |x| maximum over contiguous rows: x is [n_rows, row_len] row-major and
 *   amax_slots[r % n_channels] = max(., max_j |x[r, j]|).
 * n_channels == n_rows gives per-row (per-output-channel, axis=0) and per-block amax
 * (reduce_block_amax, core_utils.py:43-89; static block quant _amax [n_blocks,1],
 * nn/modules/tensor_quantizer.py:1008-1016); n_channels < n_rows folds leading dims
 * (amax[(idx / outer) % axis_size], kernels/quantization/gemm/tensor_quant_gpu.cu:115). */
int b200q_amax_rows(const void *x, int dtype, size_t n_rows, size_t row_len, size_t n_channels,
                    float *amax_slots, b200q_stream_t stream);

/* Column-wise |x| maximum: x is [n_rows, n_cols] row-major, amax_slots[c] = max(., max_r |x[r,c]|).
 * Per-input-channel activation amax used by SmoothQuant / AWQ (axis=-1,
 * quantization/model_calib.py:1299-1305, 1513-1530). */
int b200q_amax_cols(const void *x, int dtype, size_t n_rows, size_t n_cols, float *amax_slots,
                    b200q_stream_t stream);

/* Column-wise sum of |x| (fp32 accumulation): sum_slots[c] += sum_r |x[r,c]|.
 * AWQ-lite act_scale numerator (get_act_scale, quantization/model_calib.py:1471). */
int b200q_abssum_cols(const void *x, int dtype, size_t n_rows, size_t n_cols, float *sum_slots,
                      b200q_stream_t stream);

/* Histogram of |x| (or x when take_abs == 0) with torch.histc semantics on [0, *range_max]:
 *   bin = (int)(v * nbins / range_max), bin == nbins -> nbins-1, values outside ignored;
 *   hist[bin] += 1 (fp32 counts, like histc's output dtype).
 * Replaces the abs / float() / histc chain of HistogramCalibrator.collect
 * (quantization/calib/histogram.py:77-130). range_max is a device fp32 scalar (e.g. an amax slot). */
int b200q_histogram(const void *x, int dtype, size_t n, int take_abs, const float *range_max,
                    int nbins, float *hist, b200q_stream_t stream);

/* ---- multi-tensor (pointer-array) launches -------------------------------------------------------------------
 * ONE grid over a table of tensors -- for the many ~32 MiB activations of a calibration step, so that each tensor's
 * launch ramp / tail overlaps its neighbours'.  descs: device array of n_desc entries of 5 x 64 bits
 *   { const void *x; void *y; uint64 n_units; uint64 first_cta; int64 slot; }
 * x (and y) 32-byte aligned; n_units = the tensor's 32-byte vectors (amax) / 16-element blocks (NVFP4, rows a multiple
 * of 16); first_cta = running sum of ceil(n_units / units_per_cta) with units_per_cta = 1024 (amax) / 512 (NVFP4);
 * total_ctas = that sum over all entries.  Same arithmetic as b200q_amax_per_tensor / b200q_fake_quant_nvfp4:
 * slots[slot] = max(slots[slot], max|x|);  y = nvfp4_fake_quant(x; global amax = amax_base[slot]). */
int b200q_amax_per_tensor_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, float *slots,
                                b200q_stream_t stream);
int b200q_fake_quant_nvfp4_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, const void *amax_base,
                                 int amax_dtype, b200q_stream_t stream);

/* One read of each activation for collect + fake quant, with a speculative amax and an exact fix-up:
 *   collect_fake_quant: b200q_fake_quant_nvfp4_multi (NVFP4 descs, amax = amax_base[slot], the value exported one step
 *                       earlier) that ALSO does b200q_amax_per_tensor_multi's slots[slot] = max(slots[slot], max|x|).
 *                       Where outputs share a buffer, the caller launches it twice in stream order over sub-tensor
 *                       descriptors: the second launch holds the tiles of 512 blocks that an entry writes last while
 *                       an earlier entry writes them too (ops.second_pass_tiles), so their stores land last;
 *   fixup             : then, before the export, every entry whose slot rounded to amax_dtype as b200q_amax_export
 *                       rounds it differs in bits from amax_base[slot] is fake-quantized again with that new amax over
 *                       its live blocks [live[2i], n_units) (live: device array of n_desc x 2 uint64 from
 *                       ops.live_block_ranges; live[2i] is the first block of entry i's output that no later entry
 *                       overwrites), and the pieces (device array of n_pieces x 3 int64: entry, first block, end block)
 *                       are fake-quantized again with the exported amax: the live blocks of the tiles where live
 *                       blocks of two entries meet (ops.output_tiles).  *redo_count += number of entries whose amax
 *                       changed.
 * After the export, outputs, slots and amax_base are bit-identical to collect -> export -> fake quant, provided no
 * output overlaps an input and outputs overlap only as prefixes of one buffer (same base pointer). */
int b200q_collect_fake_quant_nvfp4_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, float *slots,
                                         const void *amax_base, int amax_dtype, b200q_stream_t stream);
int b200q_fake_quant_nvfp4_multi_fixup(const void *descs, const void *live, int n_desc, int dtype,
                                       const float *slots, const void *amax_base, int amax_dtype, const void *pieces,
                                       int n_pieces, int *redo_count, b200q_stream_t stream);

/* amax search over a collected histogram (HistogramCalibrator.compute_amax, quantization/calib/histogram.py:137-343;
 * host-side NumPy / Python loops in the reference -- one CTA per candidate here).  hist: integer-valued fp32 counts.
 *   percentile: *idx_out = searchsorted(cumsum(hist / total), percentile / 100)           (:325-343; amax = edges[idx])
 *   entropy   : div_out[c] = KL divergence of candidate i = start_bin + c * stride, c < (nbins - start_bin) / stride + 1
 *               (:210-278; amax = edges[last argmin * stride + start_bin]); scratch: nbins + 1 entries each
 *   mse       : mse_out[c] = mean((fq(centers; amax = centers[i]) - centers)^2 * hist), i = start_bin + c * stride <
 *               n_centers (:281-322; num_bits 0 = FP8-E4M3; amax = centers[first argmin * stride + start_bin]) */
int b200q_hist_search_percentile(const float *hist, int nbins, double percentile, int *idx_out, b200q_stream_t stream);
int b200q_hist_search_entropy(const float *hist, int nbins, int num_quant_bins, int stride, int start_bin,
                              long long *prefix_scratch, int *nz_scratch, double *div_out, b200q_stream_t stream);
int b200q_hist_search_mse(const float *hist, const float *centers, int n_centers, int num_bits, int is_unsigned,
                          int stride, int start_bin, float *mse_out, b200q_stream_t stream);

/* Sync-free range growth for the histogram collect.  plan_state: 32 device bytes, zero-initialised --
 *   { float upper; float width; float xmax_grow; int nbins; int initialized; int overflow; int n_growths; int pad; }
 * b200q_hist_plan applies, ON THE DEVICE, the decision HistogramCalibrator.collect takes on the host
 * (calib/histogram.py:111-130) for a batch whose |x| max is *batch_amax: first batch -> range [0, x_max], nbins0 bins
 * (width = x_max / nbins0, the linspace step); later batches with x_max > upper -> nbins = ceil(x_max / width),
 * upper = last entry of arange(0, x_max + width, width).  A batch that would need more than `capacity` bins sets
 * `overflow` = 1 (the histogram buffer holds `capacity` floats), a batch that would grow a zero-width range (an
 * all-zero first batch) sets `overflow` = 2, and later launches become no-ops.
 * b200q_histogram_planned bins the batch with the planned (nbins, upper), adding into hist[0 .. nbins). */
int b200q_hist_plan(const float *batch_amax, int nbins0, int capacity, void *plan_state, b200q_stream_t stream);
int b200q_histogram_planned(const void *x, int dtype, size_t n, int take_abs, const void *plan_state,
                            float *hist, b200q_stream_t stream);
/* Both of the above in one entry point, plus the fast path for 16-bit inputs: with pattern_scratch (device
 * uint32[B200Q_HIST_SCRATCH_ELEMS], zero-initialised, owned by the caller; its first 32768 words are left zeroed
 * again, the rest is overwritten by every launch) and take_abs the streaming pass only counts the 2^15 |x| bit patterns
 * (no floating-point work per element) and a 32768-thread epilogue bins each pattern once with the same exact
 * formula.  Layout: [0, 32768) one atomic counter per pattern; then B200Q_HIST_HOT_ROWS rows of 1536 words, row c = the
 * counts CTA c found for the 1536 bf16 patterns under the top of the range (stored, not added -- no atomics).
 * plan_state == NULL: explicit (range_max, nbins) as in b200q_histogram. */
#define B200Q_HIST_HOT_ROWS 160
#define B200Q_HIST_SCRATCH_ELEMS (32768 + B200Q_HIST_HOT_ROWS * 1536)
int b200q_histogram_ex(const void *x, int dtype, size_t n, int take_abs, const float *range_max, int nbins,
                       const void *plan_state, float *hist, uint32_t *pattern_scratch, b200q_stream_t stream);

/* NVFP4 activation-headroom statistics (NVFP4ActHeadroomCalibrator.collect,
 * quantization/calib/nvfp4_act_headroom.py:116-149): per 16-element block amax b (blocks along the
 * flat tensor; the last dim must be a multiple of 16), running_max_slot = max(., b); for b > 0:
 *   idx = clamp(floor((log2(b) - log2_min) / (log2_max - log2_min) * nbins), 0, nbins - 1); hist[idx] += 1
 * hist is int64 (torch.bincount output). */
int b200q_nvfp4_block_log2_hist(const void *x, int dtype, size_t n_blocks, float log2_min,
                                float log2_max, int nbins, long long *hist,
                                float *running_max_slot, b200q_stream_t stream);

/* b200q_nvfp4_block_log2_hist over a table of tensors in ONE launch (descs: the MultiDesc table of
 * b200q_amax_per_tensor_multi with n_units = 16-element blocks and first_cta counted in tiles of 512 blocks):
 * entry i adds its counts to row slot_i of hist ([n_slots][nbins], int64) and its block amax maximum to
 * running_max[slot_i] (fp32 bits, unsigned atomic max: NaN wins as in the per-tensor call).  Entries that share a
 * slot accumulate into it.  Counts and running maxima equal those of one b200q_nvfp4_block_log2_hist call per entry.
 * No host synchronisation and no allocation (graph-capturable). */
int b200q_nvfp4_block_log2_hist_multi(const void *descs, int n_desc, size_t total_ctas, int dtype, float log2_min,
                                      float log2_max, int nbins, long long *hist, float *running_max,
                                      b200q_stream_t stream);

/* Convert fp32 amax slots to `dtype` (the reference keeps _amax in the input dtype,
 * calib/max.py:64) and/or reset slots.  dst may be NULL (reset only). */
int b200q_amax_export(const float *amax_slots, size_t n, void *dst, int dtype,
                      b200q_stream_t stream);

/* ---- (2) fake-quant forward ------------------------------------------------------------- */

/* Integer fake quant  y = clamp(rint(x * s), lo, hi) / s,  s = hi / amax  (fp32, IEEE).
 * amax[(i / outer) % n_amax]; n_amax == 1 is per-tensor.  amax < 2^-24 -> 0.
 * Replaces fake_tensor_quant / fake_tensor_quant_with_axis
 * (kernels/quantization/gemm/tensor_quant_gpu.cu:43-140, tensor_quant.cpp:63-69).
 * x == y (in place) is allowed (fake_tensor_quant_). */
int b200q_fake_quant_int(const void *x, void *y, int dtype, size_t n, const void *amax,
                         int amax_dtype, size_t n_amax, size_t outer, int num_bits,
                         int is_unsigned, int narrow_range, b200q_stream_t stream);

/* FP8-E4M3 fake quant  y = float(e4m3_rne_satfinite(x * s)) * (1/s), s = 448 / amax
 * (amax <= 2^-24 -> amax = 1); amax == NULL is a plain cast round trip.
 * Replaces fake_e4m3fy / fake_e4m3fy_with_axis
 * (kernels/quantization/gemm/tensor_quant_gpu_fp8.cu:36-107). */
int b200q_fake_quant_fp8(const void *x, void *y, int dtype, size_t n, const void *amax,
                         int amax_dtype, size_t n_amax, size_t outer, b200q_stream_t stream);
/* Same tensor layout; the scale follows the reference's eager / CPU path _fp8_eager
 * (quantization/tensor_quant.py:46-59): scale = reciprocal(safe_amax) * 448 (torch's Tensor.__rtruediv__, two
 * roundings) instead of the extension's 448.f / safe_amax.  The reference takes this path whenever amax has more
 * than one non-singleton dim (scaled_e4m3_impl :78-79, e.g. FP8 2-D 128x128 block scales) and on CPU. */
int b200q_fake_quant_fp8_eager(const void *x, void *y, int dtype, size_t n, const void *amax,
                               int amax_dtype, size_t n_amax, size_t outer, b200q_stream_t stream);

/* NVFP4 dynamic fake quant (E2M1 values, E4M3 block-16 scale, fp32 global scale).
 * x is [n_rows, row_len]; blocks of 16 run along the last dim (partial last block reads zeros).
 * Replaces dynamic_block_quantize_op -> fp4_fake_quant_block
 * (kernels/quantization/gemm/fp4_kernel_hopper.py:33-170, common/nvfp4_quant.py:33-126). */
int b200q_fake_quant_nvfp4(const void *x, void *y, int dtype, size_t n_rows, size_t row_len,
                           const void *global_amax, int amax_dtype, b200q_stream_t stream);

/* NVFP4 static fake quant: calibrated per-block amax (fp32) + global amax (fp32 scalar).
 * scale_b = amax_b / 6, optionally FP8-round-tripped against global_amax * (448/fp8_max_norm) / 6.
 * Replaces static_blockwise_fp4_fake_quant + compute_fp4_scales
 * (kernels/quantization/gemm/fp4_kernel.py:194-316). block_size must be 16. */
int b200q_fake_quant_nvfp4_static(const void *x, void *y, int dtype, size_t n_blocks,
                                  int block_size, const float *block_amax,
                                  const float *global_amax, int quantize_block_scales,
                                  float fp8_max_norm, b200q_stream_t stream);

/* ---- (3) weight quant-and-pack ---------------------------------------------------------- */

/* NVFP4 pack (NVFP4QTensor.quantize, quantization/qtensor/nvfp4_tensor.py:229-342):
 *   s2 = *global_amax / (6*448)           (written to wsf2_out if non-NULL)
 *   bs = e4m3(clamp(blockamax / (6*s2), 2^-9, 448)), blockamax==0 -> 1  -> scales_e4m3 [n_rows, row_len/block_size]
 *   code = e2m1_rne(x / (float(bs) * s2)) ; packed[r, j] = code[2j+1] << 4 | code[2j]
 * block_size: 16 (NVFP4 proper) or 32 / 64 / ... / 512 (W4A8_NVFP4_FP8 and NVFP4_MLP_WEIGHT_ONLY use 32);
 * row_len must be a multiple of it (the reference zero-pads first). */
int b200q_pack_nvfp4(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                     const float *global_amax, uint8_t *packed, uint8_t *scales_e4m3,
                     float *wsf2_out, b200q_stream_t stream);
/* Same, but the caller supplies weights_scaling_factor_2 itself (the `weights_scaling_factor_2=` argument of
 * NVFP4QTensor.quantize, nvfp4_tensor.py:262,281-282 -- what TensorQuantizer._real_quantize passes,
 * nn/modules/tensor_quantizer.py:862-871): *wsf2 is used as is. */
int b200q_pack_nvfp4_scale2(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                            const float *wsf2, uint8_t *packed, uint8_t *scales_e4m3,
                            b200q_stream_t stream);
/* Same, with calibrated per-block amax (static quantizer branch, nvfp4_tensor.py:139-161). */
int b200q_pack_nvfp4_static(const void *x, int dtype, size_t n_rows, size_t row_len, int block_size,
                            const float *block_amax, const float *global_amax,
                            float fp8_max_norm, uint8_t *packed, uint8_t *scales_e4m3,
                            float *wsf2_out, b200q_stream_t stream);
/* NVFP4 unpack/dequant: y = e2m1_value(code) * (float(scale_e4m3) * wsf2)  (nvfp4_tensor.py:344-407). */
int b200q_unpack_nvfp4(const uint8_t *packed, const uint8_t *scales_e4m3, const float *wsf2,
                       void *y, int dtype, size_t n_rows, size_t row_len, int block_size,
                       b200q_stream_t stream);

/* INT4 block-wise "compress" pack with the CUDA-extension semantics of INT4QTensor.quantize
 * (qtensor/int4_tensor.py:40-88, tensor_quant_gpu.cu:311-340): arithmetic in `dtype`,
 * scales[b] = 7 / blockamax (dtype; written to scales_out), v = clamp(x*s, -8, 7),
 * nibble = roundf(v + 8) (half away from zero), byte = first << 4 | second.
 * n must be a multiple of block_size. */
int b200q_pack_int4_blockwise(const void *x, int dtype, size_t n, int block_size, void *scales_out,
                              uint8_t *packed, b200q_stream_t stream);
/* INT4_dequantize (tensor_quant_gpu.cu:262-279): y = (nibble - 8) / scale, arithmetic in dtype. */
int b200q_unpack_int4_blockwise(const uint8_t *packed, const void *scales, int dtype, size_t n,
                                int block_size, void *y, b200q_stream_t stream);
/* INT4 export pack (pack_int4_in_uint8, export/quant_utils.py:792-833): w is [out_dim, in_dim],
 * scale [out_dim, in_dim / block] (dtype `scale_dtype`); q = clamp(rne(w / scale), -8, 7) with the
 * division carried out in the promoted dtype; packed[o/2, i] = q[o, i] & 15 | q[o+1, i] << 4. */
int b200q_pack_int4_export(const void *w, int dtype, size_t out_dim, size_t in_dim,
                           const void *scale, int scale_dtype, int block_size, uint8_t *packed,
                           b200q_stream_t stream);

/* FP8 pack (FP8QTensor.quantize / to_quantized_weight, qtensor/fp8_tensor.py:41-113,
 * export/quant_utils.py:854-866):  q = e4m3fn(round_to_dtype(x / scale[(i / outer) % n_scale])),
 * overflow -> NaN like torch's float8_e4m3fn cast.  `scale_dtype` F32 with n_scale == 1 follows
 * torch's 0-dim promotion (result rounded to `dtype` before the fp8 cast). */
int b200q_pack_fp8(const void *x, int dtype, size_t n, const void *scale, int scale_dtype,
                   size_t n_scale, size_t outer, uint8_t *q, b200q_stream_t stream);
int b200q_unpack_fp8(const uint8_t *q, const void *scale, int scale_dtype, size_t n_scale,
                     size_t outer, void *y, int dtype, size_t n, b200q_stream_t stream);
/* INT8 pack / unpack (INT8QTensor.quantize / dequantize, qtensor/int8_tensor.py:36-124):
 *   q = int8(clamp(rne(round_to_dtype(x / scale[(i / outer) % n_scale])), -128, 127)),  y = dtype(q) * dtype(scale).
 * Same scale addressing and promotion rule as the FP8 pair; a NaN quotient packs as 0. */
int b200q_pack_int8(const void *x, int dtype, size_t n, const void *scale, int scale_dtype,
                    size_t n_scale, size_t outer, int8_t *q, b200q_stream_t stream);
int b200q_unpack_int8(const int8_t *q, const void *scale, int scale_dtype, size_t n_scale,
                      size_t outer, void *y, int dtype, size_t n, b200q_stream_t stream);

/* Signed max / min / sum for the affine-bias calibrator (compute_maxmin / compute_mean_bias,
 * quantization/calib/bias.py:25-76; BiasCalibrator.collect :113-149).  x is viewed as
 * [n_outer, n_groups, rows_per_group, n_cols] (contiguous); n_outer and rows_per_group are reduced,
 * slot index = group * n_cols + column (the [B, H, T, C] -> [1, H, 1, C] shape of `bias: {-2, -4}`).
 * Slots are RUNNING fp32 accumulators (initialise max to -inf, min to +inf, sum to 0); any may be NULL.
 * NaN elements are ignored by max / min. */
int b200q_reduce_keep(const void *x, int dtype, size_t n_outer, size_t n_groups, size_t rows_per_group,
                      size_t n_cols, float *max_slots, float *min_slots, float *sum_slots,
                      b200q_stream_t stream);

/* NF4 quant-and-pack (NF4QTensor.quantize, quantization/qtensor/nf4_tensor.py:74-127 + NF4_quantize_kernel,
 * kernels/quantization/gemm/tensor_quant_gpu.cu:198-260): flat blocks of block_size over n elements;
 * scale = block |x| max (tensor dtype), v = T(x / scale), code = index of the nearest of the 16 NF4 table
 * values (first minimum), byte = code[2i] << 4 | code[2i+1].  scales_in != NULL: use the given per-block
 * scales (the extension's NF4_quantize(input, scales, block_size)); else they are computed and written to
 * scales_out (n / block_size entries, tensor dtype). */
int b200q_pack_nf4(const void *x, int dtype, size_t n, int block_size, const void *scales_in,
                   void *scales_out, uint8_t *packed, b200q_stream_t stream);
/* NF4_dequantize (tensor_quant_gpu.cu:146-196): y[2k], y[2k+1] = bf16(bf16(LUT[hi / lo nibble]) *
 * bf16(scales[2k / block_size])); the output is always bfloat16 (2 * n_bytes elements). */
int b200q_unpack_nf4(const uint8_t *packed, const void *scales, int scales_dtype, size_t n_bytes,
                     int block_size, void *y_bf16, b200q_stream_t stream);

/* ---- MX formats: power-of-two (E8M0) scale per block ---------------------------------------- */

/* element formats, numbered like `enum class Types` of the reference extension
 * (kernels/quantization/gemm/tensor_quant_mx.h:40, exported by tensor_quant_mx.cu:401-411) */
typedef enum {
  B200Q_MX_E4M3 = 0, B200Q_MX_E5M2 = 1, B200Q_MX_INT8 = 2, B200Q_MX_E0M3 = 3, B200Q_MX_E1M2 = 4,
  B200Q_MX_E3M0 = 5, B200Q_MX_E2M1 = 6, B200Q_MX_E3M2 = 7, B200Q_MX_E2M3 = 8, B200Q_MX_E8M0 = 9
} b200q_mx_format;

/* MX fake quant -- replaces cuda_ext_mx.fused_amax_convert(inputs, block_size, format, Types.E8M0)
 * (kernels/quantization/gemm/tensor_quant_mx.cu:320-366, kernel :240-291; reached from
 * _dynamic_block_quantize_impl, quantization/tensor_quant.py:157-195, for MXFP8 / MXFP6 / MXFP4 /
 * MXINT8).  x is [n_rows, row_len]; blocks of block_size (8, 16 or 32) run along the row, a ragged
 * tail block is zero padded.  Per block: amax (NaN ignored); amax 0 / inf / NaN -> scale 1; else
 * unscale = 2^ceil(log2(amax / format_max)) from one IEEE division (:103-131);
 * y = sign(x) * round_to_format(|x| / unscale) * unscale  (:36-54).  y may alias x. */
int b200q_fake_quant_mx(const void *x, void *y, int dtype, size_t n_rows, size_t row_len,
                        int block_size, int elem_format, b200q_stream_t stream);

/* MXFP8 quant-and-pack (MXFP8QTensor.quantize / quantize_with_scale,
 * quantization/qtensor/mxfp8_tensor.py:150-215): block 32 along the row (zero padded),
 * scale byte = clamp(ceil(log2(amax / 448)), -127, 127) + 127 (amax <= 0 or NaN -> 0),
 * q = e4m3fn(clamp(x * 2^(127 - byte), +-448)).  q: [n_rows, row_len] bytes, scales:
 * [n_rows, ceil(row_len / 32)].  scale_in != NULL: use the given scale bytes (scale_out unused). */
int b200q_pack_mxfp8(const void *x, int dtype, size_t n_rows, size_t row_len, const uint8_t *scale_in,
                     uint8_t *q, uint8_t *scale_out, b200q_stream_t stream);
/* MXFP8QTensor.dequantize (mxfp8_tensor.py:217-262): y = T(float(q) * 2^(byte - 127)). */
int b200q_unpack_mxfp8(const uint8_t *q, const uint8_t *scale, size_t n_rows, size_t row_len, void *y,
                       int dtype, b200q_stream_t stream);

/* MXFP4 quant-and-pack (MXFP4QTensor.quantize, quantization/qtensor/mxfp4_tensor.py:37-83): flat
 * blocks of block_size; scale byte = ceil(max(log2(amax / 6), -127)) + 127; y = x / 2^e;
 * code = (y > 0 ? 0 : 8) + #{E2M1 bounds < |y|} (zeros -> 8, exact ties round down);
 * byte = code[2i+1] << 4 | code[2i].  q: n_blocks * block_size / 2 bytes, scale_out: n_blocks. */
int b200q_pack_mxfp4(const void *x, int dtype, size_t n_blocks, int block_size, uint8_t *q,
                     uint8_t *scale_out, b200q_stream_t stream);
/* MXFP4QTensor.dequantize (mxfp4_tensor.py:85-144); code 8 decodes to -0.0. */
int b200q_unpack_mxfp4(const uint8_t *q, const uint8_t *scale, size_t n_blocks, int block_size, void *y,
                       int dtype, b200q_stream_t stream);

/* host scalar: cuda_ext_mx.convert_to_exmy(x, format) (tensor_quant_mx.cu:399-400 ->
 * convert_to_types, tensor_quant_mx.h:163-190).  No device work. */
float b200q_convert_to_exmy(float x, int format);

/* ---- scale searches (AWQ-lite / SmoothQuant / MSE) -------------------------------------- */

/* y = x * scale[c]  (c = column) -- pre_quant_scale multiply (tensor_quantizer.py:1143-1144). */
int b200q_scale_cols(const void *x, void *y, int dtype, size_t n_rows, size_t n_cols,
                     const void *scale, int scale_dtype, b200q_stream_t stream);

/* AWQ-lite inner step fused into ONE pass over W (model_calib.py:1513-1560):
 *   y[r, c] = fakequant_int_block( W[r, c] * s[c] )  with dynamic per-block (block_size along c)
 *   amax taken on the scaled values in `dtype` precision, INT num_bits, narrow_range per flag.
 * Replaces weight * pre_quant_scale -> reduce_amax per block -> fake_tensor_quant_with_axis. */
int b200q_awq_scale_fake_quant(const void *w, void *y, int dtype, size_t n_rows, size_t n_cols,
                               const void *col_scale, int scale_dtype, int block_size,
                               int num_bits, int narrow_range, b200q_stream_t stream);

/* AWQ-lite weight_scale (get_weight_scale, model_calib.py:1453-1469):
 *   out[c] = mean_r( |W[r,c]| / (blockamax(r, c/block) + tiny) )   accumulated as fp32 sums in
 *   sum_slots[c]; the caller divides by n_rows. */
int b200q_awq_weight_scale_sums(const void *w, int dtype, size_t n_rows, size_t n_cols,
                                int block_size, float *sum_slots, b200q_stream_t stream);

/* MSE amax search in one pass (MseCalibrator.collect, quantization/calib/mse.py:84-119):
 * for each candidate k: loss[k] (+)= sum_i (fq(x_i; amax0 * mult[k]) - x_i)^2  (fp64 accumulators),
 * integer or FP8 (num_bits == 0 -> E4M3) fake quant, per-tensor amax0. */
int b200q_mse_sweep(const void *x, int dtype, size_t n, const float *amax0, const float *mult,
                    int n_cand, int num_bits, int is_unsigned, int narrow_range, double *loss,
                    b200q_stream_t stream);

/* Same per row (per-channel weights: x viewed as [n_rows, row_len], amax0[n_rows] fp32 holding values of the
 * amax dtype): loss[k * n_rows + r] += sum_j (fq(x[r,j]; amax_k(r)) - x[r,j])^2 in fp32, with
 * amax_k(r) = round_A(amax0[r] * m_k), A = cand_dtype (the dtype of the quantizer's _amax buffer:
 * MseCalibrator._compute_candidate_amax, calib/mse.py:80-84, multiplies [R,1] amax by a 0-dim fp32 candidate,
 * which torch evaluates in the amax dtype); m_k = round_A(mult[k]) if round_mult (torch on CUDA) else mult[k]
 * (torch on CPU). */
int b200q_mse_sweep_rows(const void *x, int dtype, size_t n_rows, size_t row_len, const float *amax0,
                         const float *mult, int n_cand, int cand_dtype, int round_mult, int num_bits,
                         int is_unsigned, int narrow_range, float *loss, b200q_stream_t stream);

/* NVFP4 per-block FP8-scale sweep (nvfp4_fp8_scale_sweep,
 * kernels/quantization/gemm/nvfp4_fp8_sweep.py:59-160): for each 16-block pick the FP8 scale
 * candidate c (126 positive finite e4m3 values / 448) minimising sum (|w| - q(|w|; s) )^2 with
 * s = c * global_amax / 6; best_amax[b] = global_amax * c (first minimum wins). */
int b200q_nvfp4_fp8_scale_sweep(const void *w, int dtype, size_t n_blocks,
                                const float *global_amax, float *best_amax,
                                b200q_stream_t stream);
/* Same with caller-supplied candidates c[n_cand] (<= 128) instead of e4m3 / 448 by IEEE division: torch on CUDA
 * evaluates `fp8_values / 448.0` (_fp8_scale_candidates.py:28-33) as a multiply by fl(1 / 448), one ulp different for
 * about half of the candidates -- pass that tensor to reproduce a GPU run of the reference. */
int b200q_nvfp4_fp8_scale_sweep_ex(const void *w, int dtype, size_t n_blocks, const float *global_amax,
                                   const float *cand, int n_cand, float *best_amax, b200q_stream_t stream);
/* Hessian-weighted sweep (nvfp4_fp8_scale_sweep_hessian, nvfp4_fp8_sweep.py:174-290; local_hessian_calibrate,
 * model_calib.py:1005): w is [cout, n_cin_blocks * 16]; for block (row, j) pick the candidate k minimising
 * dw^T H_j dw with dw = w - nvfp4_quant(w; block scale cand_scales[k]); best_amax[row * n_cin_blocks + j] =
 * cand_amaxes[k].  hessian: fp32 [n_cin_blocks, 16, 16].  First minimum wins. */
int b200q_nvfp4_fp8_scale_sweep_hessian(const void *w, int dtype, size_t cout, size_t n_cin_blocks,
                                        const float *cand_scales, const float *cand_amaxes, int n_cand,
                                        const float *hessian, float *best_amax, b200q_stream_t stream);
/* Static NVFP4 per-block multiplier search (MseCalibrator on the blocked weight, calib/mse.py:84-172; the
 * Four-Over-Six preset is mult = {1.0, 1.5} at fp8_max_norm 256): w is [n_blocks, 16]; for block b and candidate k,
 * loss[k, b] = sum_e (x_e - fq(x_e; amax0[b] * mult[k]))^2 with x the fp32 widening of w and fq the static NVFP4 fake
 * quant (as b200q_fake_quant_nvfp4_static with quantized block scales at fp8_max_norm) with an fp32 output; the
 * difference and the square are each rounded, and the 16 squares are summed in the order of ATen's CUDA
 * sum(dim=1).  best_amax[b] = amax0[b] * mult[k*] in fp32, k* = torch.argmin over k (first NaN, else first minimum).
 * loss_out (nullable): [n_cand, n_blocks] fp32.  1 <= n_cand <= 128. */
int b200q_nvfp4_static_mse_sweep(const void *w, int dtype, size_t n_blocks, const float *amax0,
                                 const float *global_amax, const float *mult, int n_cand, float fp8_max_norm,
                                 float *best_amax, float *loss_out, b200q_stream_t stream);

/* ---- (4) input rotation (normalized Hadamard transform) --------------------------------- */

/* Normalized fast Walsh-Hadamard transform over contiguous blocks of block_size = 2^k elements (k = 0..15) along
 * the last dim of x [n_rows, row_len] (row_len % block_size == 0).  Per block: widen to fp32; stages s = 0..k-1 in
 * ascending order, each mapping the pair (i, i | 2^s) with bit s of i clear to (a + b, a - b) with separate fp32
 * round-to-nearest adds; one multiply by fl32(block_size^-0.5); one RNE rounding to dtype.  y must not alias x.
 * amax_slot (may be null): amax_slot[0] = max(amax_slot[0], max |y|) over the rounded outputs, with the rule of
 * b200q_amax_per_tensor (NaN propagates) -- the collect of a per-tensor max calibrator of the rotated input.
 * Replaces fast_hadamard_transform.hadamard_transform(x.reshape(-1, row_len / block_size, block_size),
 * scale=block_size ** -0.5) as called by normalized_hadamard_transform (quantization/nn/functional.py:81-138). */
int b200q_hadamard(const void *x, void *y, int dtype, size_t n_rows, size_t row_len, size_t block_size,
                   float *amax_slot, b200q_stream_t stream);
/* y = fake_quant_nvfp4(hadamard(x)) (rotate_back = 0) or hadamard(fake_quant_nvfp4(hadamard(x))) (rotate_back = 1)
 * in one pass, bit-identical to those calls of b200q_hadamard and b200q_fake_quant_nvfp4: the rotated NVFP4
 * quantizer of TensorQuantizer.forward (quantization/nn/modules/tensor_quantizer.py:1146-1219).
 * row_len % 16 == 0 and row_len % block_size == 0; global_amax as in b200q_fake_quant_nvfp4. */
int b200q_fake_quant_nvfp4_rotated(const void *x, void *y, int dtype, size_t n_rows, size_t row_len,
                                   size_t block_size, int rotate_back, const void *global_amax, int amax_dtype,
                                   b200q_stream_t stream);

/* ---- (5) GPTQ weight calibration ------------------------------------------------------------ */

/* The column loop of one GPTQ block (gptq_blockwise_update, quantization/utils/calib_utils.py:241-276) on the fp32
 * working matrix.  w: [rows, ldw] fp32, w[0] is the block's first column (global column col0); its nb <= 128 columns
 * are replaced by the fake-quantized values.  u: [nb, ldu] fp32, the block of the upper Cholesky factor of the
 * inverse Hessian (upper triangle read).  e: [rows, nb] fp32 out, the scaled errors.  For i = 0 .. nb-1:
 *   q = Q(w_i); w_i := q; err = (w_i - q) / u[i,i]; w_j = w_j + fl(-err * u[i,j]) for j >= i; e[:, i] = err
 * (the product rounded, then added: the arithmetic of ATen's CUDA addr_).  Q by fmt:
 *   0 integer (num_bits, is_unsigned, narrow_range; b200q_fake_quant_int), 1 FP8-E4M3 (448 / amax;
 *   b200q_fake_quant_fp8): amax[row * amax_row_stride + (col0 + c) / amax_col_block] in amax_dtype
 *   (per tensor: stride 0 and a column block beyond the matrix; per row: stride 1);
 *   2 NVFP4 static (b200q_fake_quant_nvfp4_static, fp8_max_norm 448): fp32 block amax indexed the same way with
 *   amax_col_block 16, fp32 global_amax[0];
 *   3 NVFP4 dynamic (b200q_fake_quant_nvfp4): amax[0] is the per-tensor amax, the 16-element block amax is taken
 *   over the current working values at every column.
 * NVFP4 needs nb % 16 == 0 and col0 % 16 == 0.  No NaN / inf special case beyond the quantizers' own rules. */
int b200q_gptq_block(float *w, size_t ldw, size_t rows, int nb, const float *u, size_t ldu, float *e, int fmt,
                     const void *amax, int amax_dtype, size_t amax_row_stride, size_t amax_col_block, size_t col0,
                     int num_bits, int is_unsigned, int narrow_range, const float *global_amax,
                     b200q_stream_t stream);

/* ---- self tests (device-side numerics used by tests/, not by the product path) ----------- */
/* Checks the hoisted-reciprocal exact division against div.rn.f32 on n pseudo-random pairs
 * (seeded); returns the number of mismatches in *mismatches_host. */
int b200q_selftest_fastdiv(uint64_t seed, size_t n, unsigned long long *mismatches_host);
/* Checks the branch-free E2M1 rounding of the fake-quant kernels against the reference's compare chain on every
 * non-negative fp32 bit pattern (finite, +inf and NaN); returns the number of mismatches in *mismatches_host. */
int b200q_selftest_e2m1_round(unsigned long long *mismatches_host);

#ifdef __cplusplus
}
#endif
#endif /* B200QUANT_H_ */
