"""De-duplication of quantizer work on IDENTICAL input tensors (SURVEY.md 8(f4), VERDICT r01 "algorithmic waste").

In a decoder layer q/k/v read one tensor and gate/up read one tensor, yet each of the 7 linears owns an input quantizer
with the same configuration: the reference (and a naive engine) runs 7 calibration collects and 7 fake quants per layer
where 4 distinct tensors exist -- 43 % of the activation traffic.  Here the first quantizer that sees a tensor object (the
*leader*) does the work; a later quantizer with the same configuration that is handed the very same tensor object

  * during calibration shares the leader's calibrator (one statistic, so the loaded ``_amax`` buffers are aliased), and
    skips its collect;
  * during the quantized forward returns the leader's fake-quant output when it reads the same ``_amax`` storage.

Identity is by Python object (checked through a weak reference, like the reference's own tensor-keyed shared-input
discovery for export, unified_export_hf.py:279-349) plus the tensor's version counter: no address reuse hazards, nothing
kept alive.
Results are bit-identical to the undeduplicated run; ``TensorQuantizer.share_identical_inputs = False`` turns it off.
"""

from __future__ import annotations

import weakref

import torch

# id(tensor) -> (weakref to the tensor, {(signature, version): entry}).  A WeakKeyDictionary cannot hold tensors (its
# key comparison calls Tensor.__eq__); identity is checked through the weak reference instead, and the weakref
# callback drops the record when the tensor dies, so a recycled id can never alias a dead tensor's record.
_REGISTRY: dict = {}
stats = {"collect_skipped": 0, "fake_quant_reused": 0}


def _records(x, create: bool):
    k = id(x)
    rec = _REGISTRY.get(k)
    if rec is not None and rec[0]() is x:
        return rec[1]
    if not create:
        return None

    def _drop(ref, k=k):
        cur = _REGISTRY.get(k)
        if cur is not None and cur[0] is ref:
            del _REGISTRY[k]

    d: dict = {}
    _REGISTRY[k] = (weakref.ref(x, _drop), d)
    return d


def signature(q) -> tuple:
    bs = q._block_sizes
    return (str(q._num_bits), str(q._axis), None if bs is None else tuple(sorted((str(k), str(v)) for k, v in bs.items())),
            q._unsigned, q._narrow_range, q._dynamic, q._fake_quant, type(q._calibrator).__name__,
            (q.rotate_is_enabled, q.rotate_back_is_enabled, q.rotate_block_size))


def eligible(q, x) -> bool:
    return (getattr(q, "_is_input_quantizer", False) and type(q).share_identical_inputs and not torch.is_grad_enabled()
            and x.is_cuda and not hasattr(q, "_pre_quant_scale") and q._bias is None and not q.is_static_block_quant)


def _entry(x, q, create):
    per_tensor = _records(x, create)
    if per_tensor is None:
        return None
    key = (signature(q), x._version)
    e = per_tensor.get(key)
    if e is None and create:
        e = {"leader": weakref.ref(q), "collected": False, "outputs": {}}
        per_tensor[key] = e
    return e


def collect_once(q, x) -> bool:
    """True if ``q`` has to collect ``x`` itself; False if a sibling with the same configuration already collected this
    very tensor (``q`` then shares that sibling's calibrator)."""
    e = _entry(x, q, create=True)
    leader = e["leader"]()
    if leader is None or leader is q or not e["collected"]:
        e["leader"], e["collected"] = weakref.ref(q), True
        return True
    if q._calibrator is not leader._calibrator:
        q._calibrator = leader._calibrator          # one statistic for the group from now on
        leader._calibrator._b200_shared = True
    stats["collect_skipped"] += 1
    return False


def cached_output(q, x):
    e = _entry(x, q, create=False)
    if e is None or not hasattr(q, "_amax"):
        return None
    out = e["outputs"].get(q._amax.data_ptr())
    if out is not None:
        stats["fake_quant_reused"] += 1
    return out


def store_output(q, x, out):
    if hasattr(q, "_amax"):
        _entry(x, q, create=True)["outputs"][q._amax.data_ptr()] = out
