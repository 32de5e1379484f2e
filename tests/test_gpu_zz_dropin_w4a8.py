"""W4A8_AWQ_BETA_CFG through the drop-in: the reference's SequentialQuantizer (INT4 block-128 then FP8 per-tensor on the
weight, tensor_quantizer.py:1797) with every member on the b200 backend / calibrator, awq_lite on top.  Kept in its
own, last-sorted file; its configuration half runs on CPU in tests/test_dropin_cpu.py.  This repo's own quantize() has
no W4A8_AWQ_BETA_CFG preset, so there is no engine arm to hold against stored reference results: the test needs the
reference installed."""
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "_dropin_helpers", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_modelopt_dropin.py"))
d = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(d)


@pytest.fixture(scope="module")
def env():
    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("baseline/_ref not populated (run __graft_entry__.build() where /root/reference exists)")
    mtq = ref_env.activate()
    ref_env.use_prebuilt_extensions()
    from model_optimizer_b200 import backend

    return d.Env(mtq, backend)


def test_w4a8_awq_sequential_quantizer(env):
    """W4A8_AWQ_BETA_CFG: the reference's SequentialQuantizer (INT4 block-128 then FP8 per-tensor on the weight,
    tensor_quantizer.py:1797) with every member on the b200 backend / calibrator, awq_lite on top."""
    stock, mine, st = d.run_pair(env, "W4A8_AWQ_BETA_CFG")
    seq = [n for n, m in mine.named_modules() if type(m).__name__ == "SequentialQuantizer"]
    assert seq, "the preset did not create SequentialQuantizers"
    n = d.assert_buffers_equal(env, stock, mine, "W4A8_AWQ_BETA_CFG")
    for n0, p0, p1 in d.case_params(env, stock, mine, "W4A8_AWQ_BETA_CFG"):
        assert torch.equal(p0, p1), n0
    env[1].stats.clear()
    bad, tot = d.per_quantizer_outputs(env, stock, mine, True, "W4A8_AWQ_BETA_CFG")
    rel = d.compare_outputs(env, stock, mine, True, "W4A8_AWQ_BETA_CFG")
    assert env[1].stats.get("entrypoint", 0) > 0, dict(env[1].stats)
    assert n > 0 and tot > 0 and rel == 0.0
