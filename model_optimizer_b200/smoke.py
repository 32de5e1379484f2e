"""smoke(): one small invocation of the hot path on cuda:0, checked against the CPU oracle
(the oracle is test infrastructure; this is one of the few places allowed to import it)."""

from __future__ import annotations

import os
import sys

import numpy as np
import torch


def run():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from oracle import oracle_np as o

    from . import ops
    from .config import get_preset
    from .model_quant import quantize

    if not torch.cuda.is_available():
        raise RuntimeError("smoke() needs cuda:0 (no CPU fallback)")
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(256, 1024, device="cuda", generator=g).to(torch.bfloat16)
    xh = x.float().cpu().numpy()

    # (1) calibration collect
    slot = torch.zeros(1, dtype=torch.float32, device="cuda")
    ops.amax_per_tensor_(slot, x)
    assert float(slot) == float(o.reduce_amax(xh)), "amax mismatch"
    # (2) fake-quant forward: NVFP4, FP8, INT8
    gam = o.reduce_amax(xh)
    for name, got, ref in (
        ("nvfp4", ops.fake_quant_nvfp4(x, slot), o.fake_quant_nvfp4(xh, gam, "bf16")),
        ("fp8", ops.fake_quant_fp8(x, slot), o.fake_quant_fp8(xh, gam, 1, "bf16")),
        ("int8", ops.fake_quant_int(x, slot, 8, False, False), o.fake_quant_int(xh, gam, 8, False, False, 1, "bf16")),
    ):
        a = got.float().cpu().numpy()
        assert np.array_equal(a.view(np.uint32), ref.view(np.uint32)), f"{name} fake quant mismatch"
    # (3) weight quant-and-pack
    packed, scales, wsf2 = ops.pack_nvfp4(x, slot)
    p, s, s2 = o.pack_nvfp4(xh)
    assert np.array_equal(packed.cpu().numpy(), p) and np.array_equal(scales.view(torch.uint8).cpu().numpy(), s)
    pi, si = ops.pack_int4_blockwise(x, 128)
    rp, rs = o.pack_int4_blockwise_cuda(xh, 128, "bf16")
    assert np.array_equal(pi.cpu().numpy(), rp), "int4 pack mismatch"
    # (4) the API surface: mtq.quantize-style PTQ of a tiny MLP with the NVFP4 preset
    model = torch.nn.Sequential(torch.nn.Linear(1024, 512), torch.nn.GELU(), torch.nn.Linear(512, 256)).to(torch.bfloat16).cuda()
    with torch.no_grad():
        quantize(model, get_preset("NVFP4_DEFAULT_CFG"), lambda m: m(x))
        y = model(x)
    assert torch.isfinite(y).all()
    assert float(model[0].input_quantizer.amax) == float(gam)
    # (5) round-2 kernels: grouped (pointer-array) launches, histogram collect + GPU amax search, per-row MSE sweep
    xs = [x, (x * 0.5).contiguous()]
    slots = torch.zeros(2, dtype=torch.float32, device="cuda")
    ops.amax_per_tensor_multi_(slots, ops.TensorTable(xs, unit="vec32"))
    assert float(slots[0]) == float(gam) and float(slots[1]) == float(o.reduce_amax(xh * 0.5))
    ys = [torch.empty_like(t) for t in xs]
    ops.fake_quant_nvfp4_multi(ops.TensorTable(xs, None, ys, "block16"), slots)
    assert torch.equal(ys[0], ops.fake_quant_nvfp4(x, slot))
    # fused collect + fake quant from reset (speculative amax 0: both entries are redone) + fix-up + export
    slots2, amax2 = torch.zeros_like(slots), torch.zeros_like(slots)
    ys2, redo = [torch.empty_like(t) for t in xs], torch.zeros(1, dtype=torch.int32, device="cuda")
    t_fused = ops.TensorTable(xs, None, ys2, "block16", fused=True)
    ops.collect_fake_quant_nvfp4_multi(t_fused, slots2, amax2)
    ops.fake_quant_nvfp4_multi_fixup(t_fused, slots2, amax2, redo)
    amax2.copy_(slots2)
    assert torch.equal(slots2, slots) and int(redo) == 2, "fused collect mismatch"
    assert all(torch.equal(a, b) for a, b in zip(ys2, ys)), "fused fake quant mismatch"
    # two entries sharing one output buffer: the second one's stores must be what the buffer keeps
    yb = torch.empty_like(x)
    t_ring = ops.TensorTable(xs, None, [yb, yb], "block16", fused=True)
    ops.collect_fake_quant_nvfp4_multi(t_ring, slots2, amax2)
    ops.fake_quant_nvfp4_multi_fixup(t_ring, slots2, amax2, redo)
    assert torch.equal(yb, ys[1]) and int(redo) == 2, "fused fake quant into a shared buffer mismatch"
    from .calib import HistogramCalibrator

    hc = HistogramCalibrator(8, None, False, num_bins=512)
    hc.collect(x)
    ref_h = o.HistogramCalibrator(512)
    ref_h.collect(xh)
    assert np.array_equal(hc._calib_hist.cpu().numpy(), ref_h.hist), "histogram mismatch"
    for method, want in (("percentile", o.hist_amax_percentile(ref_h.hist, ref_h.edges, 99.99)),
                         ("mse", o.hist_amax_mse(ref_h.hist, ref_h.edges, 8, False, 1, 128)),
                         ("entropy", o.hist_amax_entropy(ref_h.hist, ref_h.edges, 8, False, 4, 128))):
        kw = {"stride": 4} if method == "entropy" else {}
        assert float(hc.compute_amax(method, **kw)) == float(want), f"histogram {method} search mismatch"
    a0 = o.round_bf16(np.abs(xh).max(axis=1, keepdims=True))
    mult = torch.linspace(0.25, 4.0, 39, device="cuda")
    loss = torch.zeros(39, 256, dtype=torch.float32, device="cuda")
    ops.mse_sweep_rows_(loss, x, torch.from_numpy(a0).cuda().to(torch.bfloat16).reshape(-1), mult, 8, False, False)
    ref_l = o.mse_sweep_losses_rows(xh, a0, mult.cpu().numpy(), 8, False, False, "bf16", round_mult=True)
    assert np.allclose(loss.cpu().numpy(), ref_l, rtol=1e-5), "per-row MSE sweep mismatch"
    # (6) input rotation: the transform (with its folded collect), its round trip and the fused rotated NVFP4 pass
    from tools.hadamard_oracle import hadamard as had_ref

    rs = torch.zeros(1, dtype=torch.float32, device="cuda")
    r = ops.hadamard(x, 128, rs)
    assert np.array_equal(r.float().cpu().numpy().view(np.uint32), had_ref(xh, 128, "bf16").view(np.uint32)), \
        "hadamard mismatch"
    assert float(rs) == float(o.reduce_amax(r.float().cpu().numpy())), "rotated collect mismatch"
    rr = ops.hadamard(r, 128)
    assert float((rr.float() - x.float()).abs().max()) <= 2 ** -6 * float(x.float().abs().max()), "rotation round trip"
    fused = ops.fake_quant_nvfp4_rotated(x, 128, rs.to(torch.bfloat16), True)
    assert torch.equal(fused, ops.hadamard(ops.fake_quant_nvfp4(r, rs.to(torch.bfloat16)), 128)), "rotated NVFP4 mismatch"
    # (7) one GPTQ block (NVFP4 dynamic weights, 128 columns) against the C oracle
    from tools import gptq_oracle

    gw = x[:64, :128].float().contiguous() * 0.05
    gx = torch.randn(512, 128, device="cuda", generator=g, dtype=torch.float64)
    gu = torch.linalg.cholesky(torch.cholesky_inverse(torch.linalg.cholesky(gx.T @ gx / 512)), upper=True).float()
    gamax = gw.abs().amax().reshape(1).to(torch.bfloat16)
    want_w, want_e = gptq_oracle.gptq_block(gw.cpu().numpy(), gu.cpu().numpy(), ops.GPTQ_NVFP4_DYNAMIC,
                                            gamax.float().cpu().numpy())
    ge = ops.gptq_block_update(gw, gu, ops.GPTQ_NVFP4_DYNAMIC, gamax)
    assert np.array_equal(gw.cpu().numpy().view(np.uint32), want_w.view(np.uint32)), "GPTQ block weights mismatch"
    assert np.array_equal(ge.cpu().numpy().view(np.uint32), want_e.view(np.uint32)), "GPTQ block errors mismatch"
    # (8) the Four-Over-Six block search (static NVFP4 at 256, multipliers {1.0, 1.5}) against the oracle
    from tools import nvfp4_mse_oracle

    fa0 = o.round_bf16(np.abs(xh).reshape(-1, 16).max(axis=1))
    fg = np.float32(fa0.max())
    fmult = torch.linspace(1.0, 1.5, 2, device="cuda")
    fbest = ops.nvfp4_static_mse_sweep(x, torch.from_numpy(fa0).cuda(), torch.tensor([fg], device="cuda"), fmult, 256.0)
    fwant, _, _ = nvfp4_mse_oracle.search(xh, fa0, fg, fmult.cpu().numpy(), 256.0, "cuda")
    assert np.array_equal(fbest.cpu().numpy().view(np.uint32), fwant.view(np.uint32)), "Four-Over-Six search mismatch"
    # (9) the grouped NVFP4 block log2 histogram against one per-tensor launch per entry (entries 0 and 2 share slot 0)
    hx = [x, (x * 1e-3).contiguous(), x[:3].contiguous()]
    hh, hm = torch.zeros(2, 512, dtype=torch.int64, device="cuda"), torch.zeros(2, dtype=torch.float32, device="cuda")
    ops.nvfp4_block_log2_hist_multi_(hh, hm, ops.TensorTable(hx, [0, 1, 0], unit="block16"))
    wh, wm = torch.zeros_like(hh), torch.zeros_like(hm)
    for t, sl in zip(hx, (0, 1, 0)):
        ops.nvfp4_block_log2_hist_(wh[sl], wm[sl:sl + 1], t)
    assert torch.equal(hh, wh) and torch.equal(hm, wm), "grouped block log2 histogram mismatch"
    torch.cuda.synchronize()
    print("smoke ok: collect / fake quant (NVFP4, FP8, INT8) / pack (NVFP4, INT4) / grouped and fused launches / histogram + "
          "amax searches / MSE sweep / Hadamard rotation / GPTQ block / Four-Over-Six search / grouped block log2 "
          "histogram match the oracle")
