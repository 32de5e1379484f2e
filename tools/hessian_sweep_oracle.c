/*
 * hessian_sweep_oracle.c -- CPU ORACLE (test infrastructure, NOT product code): the Hessian-weighted NVFP4 FP8-scale
 * sweep (b200q_nvfp4_fp8_scale_sweep_hessian; the reference: nvfp4_fp8_sweep.py:174-226) in plain C.
 *
 * Per 16-element block (row, j) of a [cout, n_cin * 16] weight, with x the fp32 widening of the weight and a = |x|:
 *   for candidate k: s = cand_scales[k], or 1 when that is 0
 *     q  = e2m1_rne_sat(fl(a / s))          IEEE division (the kernel's ExactDiv window and __fdiv_rn fallback)
 *     d  = fl(a - fl(q * s))
 *     dw = d if x >= 0 else -d              (-0.0 keeps its sign; NaN compares false and flips)
 *     h_c  = fmaf(dw[r], H[j][r][c], h_c)   r = 0 .. 15 ascending, from 0
 *     loss = fmaf(h_c, dw[c], loss)         c = 0 .. 15 ascending, from 0
 *   the winner is the first k with loss < best, best starting at +inf (Triton's rule: a NaN loss never wins; when
 *   every loss is NaN or +inf, k = 0 wins);  best_amax[row * n_cin + j] = cand_amaxes[k].
 * Every operation is one IEEE fp32 operation or one explicit fmaf: build with -ffp-contract=off.
 */
#include <math.h>
#include <stddef.h>

/* fp4_round_magnitude (common/nvfp4_quant.py:33-63): round to nearest E2M1 magnitude, ties to even, saturating at
 * 6; NaN (every comparison false) -> 6 */
static float e2m1_rne_sat(float a) {
  return a <= 0.25f ? 0.0f : a < 0.75f ? 0.5f : a <= 1.25f ? 1.0f : a < 1.75f ? 1.5f
       : a <= 2.5f ? 2.0f : a < 3.5f ? 3.0f : a <= 5.0f ? 4.0f : 6.0f;
}

/* w: [cout, n_cin * 16] fp32; hessian: [n_cin, 16, 16] fp32; best_amax: [cout * n_cin];
 * losses (may be NULL): [n_cand, cout * n_cin], the loss of every candidate for every block. */
void oracle_hessian_sweep(const float *w, size_t cout, size_t n_cin, const float *hessian, const float *cand_scales,
                          const float *cand_amaxes, int n_cand, float *best_amax, float *losses) {
  const size_t n_blocks = cout * n_cin;
  for (size_t row = 0; row < cout; ++row) {
    for (size_t j = 0; j < n_cin; ++j) {
      const size_t blk = row * n_cin + j;
      const float *x = w + blk * 16;
      const float *H = hessian + j * 256;
      float best = INFINITY;
      int best_k = 0;
      for (int k = 0; k < n_cand; ++k) {
        const float s = cand_scales[k] == 0.0f ? 1.0f : cand_scales[k];
        float dw[16];
        for (int e = 0; e < 16; ++e) {
          const float a = fabsf(x[e]);
          const float q = e2m1_rne_sat(a / s);
          const float d = a - q * s;
          dw[e] = x[e] >= 0.0f ? d : -d;
        }
        float loss = 0.0f;
        for (int c = 0; c < 16; ++c) {
          float h = 0.0f;
          for (int r = 0; r < 16; ++r) h = fmaf(dw[r], H[r * 16 + c], h);
          loss = fmaf(h, dw[c], loss);
        }
        if (losses) losses[(size_t)k * n_blocks + blk] = loss;
        if (loss < best) {
          best = loss;
          best_k = k;
        }
      }
      best_amax[blk] = cand_amaxes[best_k];
    }
  }
}
