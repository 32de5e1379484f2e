"""The Hessian-weighted NVFP4 FP8-scale sweep oracle (tools/hessian_sweep_oracle.c) and the local-Hessian accumulation,
without a GPU: against the reference's own CPU sweep and accumulator (tests/golden/ref_hessian_sweep.npz, written by
tools/gen_hessian_sweep_golden.py) and on constructed cases for the winner rule."""

import numpy as np
import pytest
import torch

from oracle import golden
from tools import hessian_sweep_oracle as hso

NEAR_TIE = 2.0 ** -20          # |L64(k1) - L64(k2)| <= NEAR_TIE * sum |dw_b H_bd dw_d|: within fp32 summation error


@pytest.fixture(scope="module")
def ref():
    return golden.load("ref_hessian_sweep")


def sweep_cases(ref):
    return sorted({k.rsplit("/", 1)[0] for k in ref.files if k.startswith("sweep/")})


def ref_candidates(ref, key):
    """The reference's candidate values: amax fl32(g * c), block scale fl32(amax / 6) (its quant_func does not round
    the scale to FP8)."""
    amax = (ref[f"{key}/cand"].astype(np.float32) * np.float32(ref[f"{key}/g"])).astype(np.float32)
    return (amax / np.float32(6)).astype(np.float32), amax


def test_oracle_vs_reference_sweep_fixture(ref):
    """The oracle's winners equal the reference's 126-step einsum sweep except at certified near-ties (< 1 %), and
    its losses are the reference's (which sums the block loss over the block's 16 elements) to fp32 summation error."""
    total = ties = 0
    for key in sweep_cases(ref):
        w, want = ref[f"{key}/w"], ref[f"{key}/best"]
        n_cin = w.shape[1] // 16
        hess = ref[f"hess/{w.shape[1]}/h_bits"].view(np.float32)
        scales, amaxes = ref_candidates(ref, key)
        assert np.all(np.diff(amaxes) > 0)
        got, losses = hso.hessian_sweep(w, hess, scales, amaxes, return_losses=True)
        k_got, k_want = np.searchsorted(amaxes, got), np.searchsorted(amaxes, want)
        assert np.array_equal(amaxes[k_got], got) and np.array_equal(amaxes[k_want], want), key
        l64, bound = hso.loss64(hso.residual(w, scales), hess, n_cin)
        b = np.arange(want.size)
        gap = np.abs(l64[k_got, b] - l64[k_want, b])
        certified = gap <= NEAR_TIE * np.maximum(bound[k_got, b], bound[k_want, b])
        off = k_got != k_want
        assert certified[off].all(), (key, np.flatnonzero(off & ~certified)[:8])
        total += want.size
        ties += int(off.sum())
        lref = ref[f"{key}/losses"].astype(np.float64)
        n = lref.shape[1]
        assert n == int(ref[f"{key}/loss_rows"]) * n_cin
        err = np.abs(16.0 * losses[:, :n].astype(np.float64) - lref)
        assert np.all(err <= 16 * 2.0 ** -18 * bound[:, :n]), (key, float(err.max()))
    print(f"hessian sweep fixture: {ties} certified near-tie blocks of {total}")
    assert ties < 0.01 * total, (ties, total)


def run(w, hess, scales, amaxes):
    best, losses = hso.hessian_sweep(np.asarray(w, np.float32).reshape(-1, np.asarray(hess).shape[0] * 16),
                                     hess, scales, amaxes, return_losses=True)
    return best, losses


E2M1 = np.array([0, 0.5, 1, 1.5, 2, 3, 4, 6] * 2, np.float32) * np.array([1, -1] * 8, np.float32)


def test_duplicate_scales_first_wins():
    """Two candidates with the same scale (so the same loss) and different amaxes: the earlier one wins."""
    s = np.float32(0.125)
    w = E2M1 * s                                                   # exact on the grid of s: loss 0
    h = np.eye(16, dtype=np.float32)[None]
    best, losses = run(w, h, [0.3, s, s, 0.01], [10.0, 20.0, 30.0, 40.0])
    assert losses[1, 0] == 0 and losses[2, 0] == 0 and losses[0, 0] > 0
    assert best[0] == 20.0
    best, _ = run(w, h, [s, s], [7.0, 8.0])
    assert best[0] == 7.0


def test_nan_loss_candidates_are_skipped():
    w = np.linspace(-1, 1, 16, dtype=np.float32)
    h = np.eye(16, dtype=np.float32)[None]
    best, losses = run(w, h, [np.nan, np.inf, 0.2, 0.05, np.nan], [1.0, 2.0, 3.0, 4.0, 5.0])
    assert np.isnan(losses[[0, 1, 4], 0]).all() and np.isfinite(losses[[2, 3], 0]).all()
    assert best[0] == (3.0 if losses[2, 0] <= losses[3, 0] else 4.0)


def test_all_nan_or_inf_losses_pick_candidate_zero():
    h = np.eye(16, dtype=np.float32)[None]
    w = np.linspace(-1, 1, 16, dtype=np.float32)
    w[3] = np.nan                                                  # a NaN weight: every loss NaN
    best, losses = run(w, h, [0.1, 0.2, 0.3], [1.0, 2.0, 3.0])
    assert np.isnan(losses).all() and best[0] == 1.0
    w = np.linspace(-1, 1, 16, dtype=np.float32)
    hinf = np.full((1, 16, 16), np.inf, np.float32)                # inf Hessian: +inf (or NaN) losses
    best, losses = run(w, hinf, [0.1, 0.2, 0.3], [1.0, 2.0, 3.0])
    assert not np.isfinite(losses).any() and best[0] == 1.0


def test_zero_hessian_block_picks_candidate_zero():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((4, 32)).astype(np.float32)
    h = np.stack([np.zeros((16, 16), np.float32), np.eye(16, dtype=np.float32)])
    scales = np.float32([0.5, 0.3, 0.2, 0.1, 0.05])
    best, losses = run(w, h, scales, scales * 6)
    assert np.all(losses[:, 0::2] == 0)
    assert np.all(best[0::2] == np.float32(3.0))                   # every loss 0: the first candidate
    assert np.array_equal(best[1::2], (scales * 6)[np.argmin(losses[:, 1::2], axis=0)])


def test_distinct_hessian_per_cin_block():
    """Each cin block has its own Hessian: the winners equal a float64 argmin with each block's own Hessian (where it
    is clear of fp32 error), and differ from a run whose Hessians are permuted."""
    rng = np.random.default_rng(1)
    n_cin, cout = 3, 64
    w = (rng.standard_normal((cout, n_cin * 16)) * (1 + 4 * (rng.random((cout, n_cin * 16)) < 0.05))).astype(np.float32)
    h = []
    for j in range(n_cin):                                         # weight a different few columns heavily per block
        d = np.full(16, 1e-3)
        d[j * 5:(j + 1) * 5] = 10.0
        a = rng.standard_normal((16, 16)) * 0.01
        h.append(np.diag(d) + a @ a.T)
    h = np.stack(h).astype(np.float32)
    g = np.abs(w).max()
    c = np.arange(1, 127, dtype=np.float32) / np.float32(126)
    amaxes = (c * np.float32(g)).astype(np.float32)
    scales = (amaxes / np.float32(6)).astype(np.float32)
    best, _ = run(w, h, scales, amaxes)
    l64, bound = hso.loss64(hso.residual(w, scales), h, n_cin)
    srt = np.sort(l64, axis=0)
    clear = (srt[1] - srt[0]) > NEAR_TIE * bound.max(axis=0)
    assert clear.mean() > 0.9
    assert np.array_equal(best[clear], amaxes[np.argmin(l64, axis=0)][clear])
    permuted, _ = run(w, h[[1, 2, 0]], scales, amaxes)
    assert (permuted != best).mean() > 0.2


def test_local_hessian_update_equals_reference_accumulator(ref):
    """model_calib._local_hessian_update over the fixture's 2-D and 3-D batches gives the reference's
    normalized_hessian() bit for bit, including an all-zero cin block."""
    from model_optimizer_b200.model_calib import _local_hessian_update

    for cin in (16, 48, 256):
        entry = [None, 0]
        i = 0
        while f"hess/{cin}/x{i}" in ref:
            _local_hessian_update(entry, torch.from_numpy(ref[f"hess/{cin}/x{i}"]), cin)
            i += 1
        assert i == 3 and entry[1] == 12 + 10 + 7
        got = (entry[0] / entry[1]).numpy()
        assert np.array_equal(got.view(np.uint32), ref[f"hess/{cin}/h_bits"]), cin
        if cin == 48:
            assert np.all(got[1] == 0) and np.all(got[0] != 0)
