"""NVFP4 activation-headroom calibration, host side: the oracle against the reference's CPU run
(tests/golden/ref_act_headroom.npz, tools/gen_act_headroom_golden.py), the config's bounds, validate-before-mutate,
and the data-parallel MAX merge of headroom amaxes over a gloo world of 2."""

import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle import oracle_np as o  # noqa: E402
from tools.gen_act_headroom_golden import CASES, DTYPES, LINEARS, net, quant_cfg  # noqa: E402

from model_optimizer_b200 import model_quant  # noqa: E402
from model_optimizer_b200.config import NVFP4ActHeadroomCalibConfig  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    return golden.load("ref_act_headroom")


def _inputs(x, lin):
    """What ``lin``'s input quantizer sees for the model input x (tools/gen_act_headroom_golden.py, Net.forward)."""
    if lin in ("q", "k"):
        return x
    if lin == "o":
        return np.maximum(x[..., :32], 0)
    if lin == "z":
        return np.zeros_like(x[..., :32])
    return None


def _pad16(x):
    r = x.shape[-1] % 16
    return x if r == 0 else np.pad(x, [(0, 0)] * (x.ndim - 1) + [(0, 16 - r)])


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_input_amax(fx, case, d):
    algo = {"anchor_percentile": 1.0, "upper_percentile": 99.99, "rho": 16384.0}
    algo.update({k: v for k, v in CASES[case][0].items() if k in algo})
    key = f"{case}/{d}"
    calib = fx[f"model/{d}/calib"]
    n_amax = 0
    for lin in LINEARS:
        p = f"{key}/{lin}.input_quantizer"
        assert bool(fx[p + ".enabled"]) and str(fx[p + ".calibrator"]) == "MaxCalibrator", p
        xs = [_inputs(x, lin) for x in calib]
        if xs[0] is None:                                    # never called: no statistic, no amax
            assert p + ".amax" not in fx, p
            continue
        hist, rmax = np.zeros(512, dtype=np.int64), np.float32(0)
        for x in xs:
            h, m = o.nvfp4_block_log2_hist(_pad16(x))
            hist, rmax = hist + h, max(rmax, np.float32(m))
        if hist.sum() == 0:                                  # all-zero input: compute_amax gives None
            assert p + ".amax" not in fx, p
            continue
        want = o.act_headroom_amax(hist, rmax, algo["anchor_percentile"], algo["upper_percentile"], algo["rho"])
        got = fx[p + ".amax"]
        assert got.shape == () and str(fx[p + ".amax_dtype"]) == "torch.float32", p
        assert np.float32(got).view(np.uint32) == np.float32(want).view(np.uint32), (p, float(got), float(want))
        n_amax += 1
    assert n_amax == 3
    # the fallback warns (twice per quantizer: finish_stats_collection computes the amax, then loads it)
    assert len(fx[f"{key}/warnings"]) == (6 if case == "small_rho" else 0)


def test_config_bounds():
    c = NVFP4ActHeadroomCalibConfig()
    assert (c.anchor_percentile, c.upper_percentile, c.rho) == (1.0, 99.99, 16384.0)
    assert c.weight_scale_algorithm == {"method": "max"}
    assert NVFP4ActHeadroomCalibConfig(anchor_percentile=100, upper_percentile=100, rho=28671.9).rho == 28671.9
    w = {"method": "local_hessian", "fp8_scale_sweep": True}
    assert NVFP4ActHeadroomCalibConfig(weight_scale_algorithm=w).weight_scale_algorithm == w
    for bad in ({"anchor_percentile": 0.0}, {"anchor_percentile": 100.5}, {"upper_percentile": 0},
                {"upper_percentile": 101}, {"rho": 0.0}, {"rho": 28672.0}, {"rho": -1.0}, {"rho": True},
                {"weight_scale_algorithm": "max"}, {"weight_scale_algorithm": {"method": "awq_lite"}},
                {"weight_scale_algorithm": {}}, {"method": "max"}):
        with pytest.raises(ValueError):
            NVFP4ActHeadroomCalibConfig(**bad)


def _prepared(cfg):
    """The mirror's model with the config applied and calibration not yet run."""
    model = net(torch.float32)
    model_quant.replace_quant_module(model)
    model_quant.set_quantizer_by_cfg(model, cfg["quant_cfg"])
    return model


def _state(model):
    return [(n, id(q._calibrator), type(q._calibrator).__name__, hasattr(q, "_amax"), q._if_calib, q._if_quant)
            for n, q in model.named_modules() if n.endswith("_quantizer")]


def test_block_size_other_than_16_leaves_model_untouched():
    cfg = quant_cfg(False, {})
    cfg["quant_cfg"][1]["cfg"]["block_sizes"][-1] = 32
    model = _prepared(cfg)
    before = _state(model)
    with pytest.raises(NotImplementedError, match="'k.input_quantizer'|'q.input_quantizer'"):
        model_quant.calibrate(model, cfg["algorithm"], lambda m: None)
    assert _state(model) == before
    with pytest.raises(ValueError, match="rho"):                 # a bad option: also refused before any change
        model_quant.calibrate(model, {"method": "nvfp4_act_headroom", "rho": 1e6}, lambda m: None)
    assert _state(model) == before


def test_no_matching_quantizer_warns():
    cfg = quant_cfg(False, {})
    cfg["quant_cfg"] = cfg["quant_cfg"][:1]                     # every quantizer disabled
    model = _prepared(cfg)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        model_quant.calibrate(model, cfg["algorithm"], None)
    assert any("no NVFP4 dynamic-block input quantizer matched" in str(w.message) for w in caught)
    assert all(type(q._calibrator).__name__ == "MaxCalibrator" for n, q in model.named_modules()
               if n.endswith("_quantizer"))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from model_optimizer_b200.calib import NVFP4ActHeadroomCalibrator
        from model_optimizer_b200.distributed import sync_headroom_amax
        from model_optimizer_b200.nn import TensorQuantizer

        cfg = {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "dynamic", "scale_bits": (4, 3)}}
        m = torch.nn.ModuleDict({n: TensorQuantizer(cfg) for n in ("a", "b", "c", "plain")})
        for n in ("a", "b", "c"):
            m[n]._calibrator = NVFP4ActHeadroomCalibrator()
        mine = {0: {"a": 2.0, "b": 5.0, "plain": 9.0}, 1: {"a": 3.0, "b": 1.0, "c": 7.0, "plain": 4.0}}[rank]
        for n, v in mine.items():
            m[n].amax = torch.tensor(v, dtype=torch.float32)
        merged = sync_headroom_amax(m)
        got = {n: (float(m[n]._amax), m[n]._amax.dtype) for n in ("a", "b", "c", "plain")}
        q.put((rank, merged, got))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_headroom_amax_max_merge_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=90) for _ in range(2))
    for p in procs:
        p.join(30)
    f32 = torch.float32
    for rank, merged, got in res:
        assert merged == 3
        # the largest per-rank scale; rank 0 adopts c; the MaxCalibrator quantizer is not part of this merge
        assert got == {"a": (3.0, f32), "b": (5.0, f32), "c": (7.0, f32), "plain": (9.0 if rank == 0 else 4.0, f32)}


def test_engine_headroom_mode_arguments():
    from model_optimizer_b200.engine import TINY, ShardedPTQEngine

    with pytest.raises(NotImplementedError):
        ShardedPTQEngine(TINY, 16, calib="nvfp4_act_headroom", world_size=2, device="cpu")
    with pytest.raises(ValueError):
        ShardedPTQEngine(TINY, 16, qformat="fp8", calib="nvfp4_act_headroom", device="cpu")
    with pytest.raises(ValueError):
        ShardedPTQEngine(TINY, 16, calib="entropy", device="cpu")
    with pytest.raises(ValueError):
        ShardedPTQEngine(TINY, 16, headroom={"rho": 4.0}, device="cpu")
