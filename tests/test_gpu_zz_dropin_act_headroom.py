"""``nvfp4_act_headroom`` through the drop-in: the stock reference ``mtq.quantize`` on the GPU, then again after
``backend.install()``, whose ``NVFP4ActHeadroomCalibrator`` rebind runs the collect on this engine.  Every ``_amax``
must be identical.  Kept in its own, last-sorted file (the rebind is process-global; ``uninstall()`` runs in a
finalizer)."""

import copy
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gen_act_headroom_golden import data, net, quant_cfg  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mtq(request):
    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("baseline/_ref not populated (run __graft_entry__.build() where /root/reference exists)")
    mod = ref_env.activate()
    ref_env.use_prebuilt_extensions()
    from model_optimizer_b200 import backend

    request.addfinalizer(backend.uninstall)
    return mod


def _amaxes(model):
    return {n: m._amax.detach().clone() for n, m in model.named_modules() if isinstance(getattr(m, "_amax", None),
                                                                                       torch.Tensor)}


def test_dropin_act_headroom_matches_stock(mtq):
    from model_optimizer_b200 import backend

    base = net(torch.bfloat16).cuda()
    calib, _ = data(torch.bfloat16)
    calib = [x.cuda() for x in calib]
    cfg = quant_cfg(False, {"anchor_percentile": 2.0})
    stock = copy.deepcopy(base)
    mtq.quantize(stock, copy.deepcopy(cfg), lambda m: [m(x) for x in calib])
    backend.install()
    backend.stats.clear()
    mine = copy.deepcopy(base)
    mtq.quantize(mine, copy.deepcopy(cfg), lambda m: [m(x) for x in calib])
    import modelopt.torch.quantization.model_calib as ref_model_calib

    assert ref_model_calib.NVFP4ActHeadroomCalibrator.__name__ == "B200NVFP4ActHeadroomCalibrator"
    assert backend.stats["calib.nvfp4_act_headroom"] > 0, dict(backend.stats)
    a, b = _amaxes(stock), _amaxes(mine)
    assert a.keys() == b.keys() and any(k.endswith("input_quantizer") for k in a)
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), (k, a[k], b[k])
    backend.uninstall()
    assert ref_model_calib.NVFP4ActHeadroomCalibrator.__name__ == "NVFP4ActHeadroomCalibrator"
