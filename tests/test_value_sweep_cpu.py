"""The value sweep's own inputs (tests/_value_sweep.py): every 16-bit pattern is there, the scale grid straddles every
window edge, and for each kernel family the built inputs reach both the fast and the slow branch, computed on the host
from the kernels' documented conditions (ExactDiv::block_ok, the NVFP4 pack's kMaxDenom and quotient bound, the FP8 /
INT8 pack's vmax <= 448 * s0 and 2^60, NF4's big)."""

import numpy as np
import pytest

import _value_sweep as vs
from oracle import oracle_np as o

F32 = np.float32
S = vs.scale_grid()


def test_every_16bit_pattern_appears():
    for dt in ("bf16", "f16"):
        v = vs.values16(dt)
        bits = o.bf16_bits(v) if dt == "bf16" else v.astype(np.float16).view(np.uint16)
        nan = np.isnan(v)
        assert np.array_equal(np.sort(bits[~nan]), np.sort(vs.patterns16()[~nan]))
        assert np.unique(vs.patterns16()).size == 65536 and nan.sum() == (254 if dt == "bf16" else 2046)
        # ±0, subnormals, ±inf and NaNs of both signs
        assert {0x0000, 0x8000, 0x0001, 0x8001}.issubset(set(vs.patterns16().tolist()))
        assert np.isposinf(v).any() and np.isneginf(v).any()
        assert (nan & (vs.patterns16() < 0x8000)).any() and (nan & (vs.patterns16() >= 0x8000)).any()


def test_fp32_domain():
    x = vs.fp32_structured()
    b = x.view(np.uint32)
    assert x.size == 6144 and np.unique(b).size == 6144
    assert set(((b >> 23) & 0xFF).tolist()) == set(range(256))
    assert np.isnan(x).any() and np.isinf(x).any() and (b == 0x80000000).any() and (b == 1).any()


@pytest.mark.parametrize("edge", vs.EDGES + vs.THRESHOLDS)
def test_scale_grid_straddles_every_edge(edge):
    e = F32(edge)
    for grid in (S, vs.coarse(S)):
        assert e in grid
        assert (grid < e).any() and grid[grid < e].max() == np.nextafter(e, F32(0))
        assert grid[grid > e].min() == np.nextafter(e, F32(np.inf))
    assert S[0] == 0 and vs.DENORM_MIN in S and vs.FLT_MAX in S
    assert F32(2.0 ** -133) in S and F32(2.0 ** 127) in S


def test_boundary_values_are_ties_and_neighbours():
    v = vs.boundary_values(F32(2.0 ** -10), vs.E2M1_T)
    t = (np.abs(v) / F32(2.0 ** -10)).astype(F32)
    for b in (0.25, 0.75, 2.5, 5.0):
        assert (t == F32(b)).any() and (t < F32(b)).any() and (t > F32(b)).any()
    assert (v < 0).sum() == (v > 0).sum()


def test_nvfp4_pack_inputs_reach_every_branch():
    """For each dtype: blocks on the fast path, blocks outside the divisor window on both sides, and fast-window
    blocks whose quotient overflows (the case the pack must route to the explicit path; fp16's largest value over
    kBlockMin cannot overflow)."""
    for dt in vs.DTYPES:
        kmax = F32(vs.K_MAX_DENOM[dt])
        seen = {"fast": False, "below": False, "above": False, "overflow": dt == "f16", "nonfinite": False}
        for w in vs.pack_wsf2_grid():
            x = vs.nvfp4_dynamic_input(dt, F32(w * F32(2688.0)))
            denom, finite = vs.nvfp4_pack_denoms(x, wsf2=w)
            fast, over = vs.nvfp4_pack_branches(x, dt, wsf2=w)
            seen["fast"] |= bool(fast.any())
            seen["below"] |= bool((finite & (denom < F32(vs.K_BLOCK_MIN))).any())
            seen["above"] |= bool((finite & (denom > kmax)).any())
            seen["overflow"] |= bool(over.any())
            seen["nonfinite"] |= bool((~finite).any())
        assert all(seen.values()), (dt, seen)
        # the clamped divisor fl(448 * w) lands on each side of kBlockMin and kMaxDenom
        d = (F32(448.0) * vs.pack_wsf2_grid()).astype(F32)
        for e in (vs.K_BLOCK_MIN, vs.K_MAX_DENOM[dt]) if dt != "f16" else (vs.K_BLOCK_MIN,):
            assert (d == np.nextafter(F32(e), F32(0))).any() and (d == np.nextafter(F32(e), F32(np.inf))).any(), (dt, e)


def test_nvfp4_pack_repro_is_an_overflow_case():
    x = np.zeros((1, 16), dtype=F32)
    x[0, 0] = -1e30
    for dt in ("bf16", "f32"):
        fast, over = vs.nvfp4_pack_branches(o.round_to(x, dt), dt, global_amax=F32(3e-9))
        assert fast[0] and over[0]


def test_nvfp4_fake_quant_inputs_reach_block_ok_both_ways():
    for dt in vs.DTYPES:
        ok = np.concatenate([vs.nvfp4_fq_block_ok(vs.nvfp4_dynamic_input(dt, g), g) for g in vs.coarse(S)])
        assert ok.any() and (~ok).any()
    # the static sweep: block scale S[r] on both sides of [kBlockMin, kBlockMax]
    assert (S < F32(vs.K_BLOCK_MIN)).any() and ((S >= F32(vs.K_BLOCK_MIN)) & (S <= F32(vs.K_BLOCK_MAX))).any()
    assert (S > F32(vs.K_BLOCK_MAX)).any()


def test_fp8_int8_pack_inputs_reach_both_paths():
    for dt in vs.DTYPES:
        sc = o.round_to(S, dt)
        sc = sc[np.isfinite(sc) & (sc > 0)]
        x = np.tile(vs.domain(dt), (sc.size, 1)) if dt != "f32" else vs.fp32_rows(sc, vs.E4M3_T)
        for int8 in (False, True):
            fast = vs.fp8_int8_pack_fast(x, sc, int8)
            assert fast.any() and (~fast).any(), (dt, int8)
        # vmax <= 448 * s0 decides alone: finite vectors inside the window on both sides of it
        vmax = np.max(np.abs(x.reshape(x.shape[0], -1, 16)), axis=-1)
        win = (sc.reshape(-1, 1) >= F32(2.0 ** -60)) & (sc.reshape(-1, 1) <= F32(2.0 ** 60)) & (vmax <= F32(2.0 ** 60))
        with np.errstate(over="ignore"):
            lim = (F32(448.0) * sc.reshape(-1, 1)).astype(F32)
        assert (win & (vmax <= lim)).any() and (win & (vmax > lim)).any(), dt


def test_nf4_inputs_reach_fast_big_and_slow():
    for dt in vs.DTYPES:
        sc = o.round_to(vs.coarse(S, 3), dt)
        sc = sc[np.isfinite(sc)]
        x = np.tile(vs.domain(dt), (sc.size, 1)) if dt != "f32" else vs.fp32_rows(sc, vs.NF4_T, 64)
        fast, big = vs.nf4_branches(x, sc, dt)
        assert (fast & ~big).any() and big.any() and (~fast).any(), dt


def test_mx_setters_cover_the_e8m0_range():
    for dt in vs.DTYPES:
        s = vs.mx_setters(dt)
        e = np.floor(np.log2(s.astype(np.float64)))
        lo = {"bf16": -133, "f16": -24, "f32": -149}[dt]
        hi = {"bf16": 127, "f16": 15, "f32": 127}[dt]
        assert e.min() == lo and e.max() == hi and np.all(np.diff(np.unique(e)) <= 3), dt
        x = vs.mx_input(dt, 32)
        assert x.shape[1] == 32
        # every setter-led block's max is its setter
        lead = x[: len(s) * 4]
        assert np.array_equal(np.max(np.abs(lead), axis=1), np.abs(lead[:, 0]))
        ex = o.e8m0_exponent_nv(np.max(np.abs(lead), axis=1), o.MX_E4M3)
        assert ex.min() <= -127 + 1 and ex.max() >= 127 - 9 if dt != "f16" else ex.max() >= 7, (dt, ex.min(), ex.max())
