"""Multi-GPU calibration: one process per GPU, layer-sharded, ONE collective.

Reference: every quantizer calls ``dist.all_reduce(MAX)`` on its own ``_amax`` buffer
(``TensorQuantizer.sync_amax_across_distributed_group``, nn/modules/tensor_quantizer.py:1377, driven by
``max_calibrate``, model_calib.py:390-495) -- ~450 one-element NCCL calls for Llama-3-8B -- and the
NVFP4 global scale of fused siblings is synchronised separately
(``SharedWeightGlobalAmaxState.sync``, utils/shared_input.py:340).

Here every calibrator's fp32 slots are views into (or are packed into) ONE flat fp32 arena and a single
``all_reduce(MAX)`` over NVLink/NVSwitch merges them.  amax >= 0, so a rank that does not own a layer
contributes zeros and MAX doubles as the all-gather of layer-sharded ownership; data-parallel replicas of
the same layer merge exactly like the reference's per-quantizer MAX.

Layer sharding: ``shard_layers(n_layers, world, rank)`` gives each rank a contiguous range of decoder
layers; quantizer statistics and weight packs of different layers are independent, so there is no
data-path collective.
"""

from __future__ import annotations

import torch
import torch.distributed as dist


def is_initialized() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def shard_layers(n_layers: int, world_size: int, rank: int) -> range:
    """Contiguous, balanced ranges: the first ``n_layers % world_size`` ranks get one extra layer."""
    base, extra = divmod(n_layers, world_size)
    start = rank * base + min(rank, extra)
    return range(start, start + base + (1 if rank < extra else 0))


class AmaxArena:
    """A flat fp32 device buffer of amax slots with named segments.

    ``register(name, n)`` on EVERY rank in the same order (the arena layout must agree across ranks,
    including segments a rank does not own); ``view(name)`` is the tensor the collect kernels write to;
    ``all_reduce()`` is the one collective.
    """

    def __init__(self, device):
        self.device = torch.device(device)
        self._segments: dict[str, tuple[int, int]] = {}
        self._size = 0
        self._buf: torch.Tensor | None = None

    def register(self, name: str, n: int = 1):
        if self._buf is not None:
            raise RuntimeError("arena is frozen")
        if name in self._segments:
            raise KeyError(f"duplicate amax segment {name}")
        self._segments[name] = (self._size, n)
        self._size += n

    def freeze(self) -> torch.Tensor:
        if self._buf is None:
            self._buf = torch.zeros(max(self._size, 1), dtype=torch.float32, device=self.device)
        return self._buf

    def view(self, name: str) -> torch.Tensor:
        off, n = self._segments[name]
        return self.freeze()[off : off + n]

    def names(self):
        return list(self._segments)

    def __len__(self):
        return self._size

    def all_reduce(self, group=None, async_op: bool = False):
        """THE collective: MAX over all ranks of the whole arena (NCCL on CUDA, gloo on CPU tests)."""
        buf = self.freeze()
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            return dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=group, async_op=async_op)
        return None


_DTYPE_CODES = {torch.float32: 1, torch.bfloat16: 2, torch.float16: 3}
_CODE_DTYPES = {v: k for k, v in _DTYPE_CODES.items()}
_MAX_DIMS = 6


def sync_calibrator_amax(model, group=None, include_weights=True) -> int:
    """Merge every MaxCalibrator's running maxima across the ranks of ``group`` with one all-reduce.

    ``group`` is the DATA-PARALLEL group (the reference syncs amax over the data-parallel group only,
    model_calib.py:121-175 ``sync_quantizer_amax_across_dp_ep``); pass ``include_weights=False`` when the ranks of the
    group hold different shards of a weight (tensor parallel), whose per-channel amax must not be merged.

    Quantizers are visited in ``named_modules`` order (identical on all ranks for the same model
    definition); calibrators that saw no data on this rank contribute zeros and adopt the merged statistic with the
    owner's keepdims shape and dtype (a header of [numel, dtype, ndim, dims...] per quantizer is MAX-reduced first).
    Returns the arena size.
    """
    from .calib import MaxCalibrator
    from .nn import TensorQuantizer

    entries = []
    device = None
    for name, q in model.named_modules():
        if not isinstance(q, TensorQuantizer) or q._disabled or not isinstance(q._calibrator, MaxCalibrator):
            continue
        if not q._if_calib and q._calibrator.slots is None:
            continue
        if not include_weights and name.endswith("weight_quantizer"):
            continue
        entries.append((name, q._calibrator))
        if q._calibrator.slots is not None:
            device = q._calibrator.slots.device
    if not entries:
        return 0
    # agree on segment sizes / shapes: a rank that never saw a layer knows neither its slot count nor its keepdims shape
    head = torch.zeros(len(entries), 3 + _MAX_DIMS, dtype=torch.int64)
    for i, (name, c) in enumerate(entries):
        if c.slots is None:
            continue
        shape = tuple(c._shape or ())
        if len(shape) > _MAX_DIMS:
            raise ValueError(f"{name}: amax of rank {len(shape)} > {_MAX_DIMS}")
        head[i, 0] = c.slots.numel()
        head[i, 1] = _DTYPE_CODES.get(c._dtype, 1)
        head[i, 2] = len(shape)
        for j, d in enumerate(shape):
            head[i, 3 + j] = d
    if dist.get_backend(group) == "nccl":
        head = head.cuda()
    dist.all_reduce(head, op=dist.ReduceOp.MAX, group=group)
    head = head.cpu().tolist()
    sizes = [h[0] for h in head]
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    arena = AmaxArena(device)
    for (name, _), n in zip(entries, sizes):
        arena.register(name, int(n))
    arena.freeze()
    for (name, c), n in zip(entries, sizes):
        if c.slots is not None and n:
            if c.slots.numel() != n:
                raise ValueError(f"{name}: {c.slots.numel()} amax slots here, {n} on another rank")
            arena.view(name).copy_(c.slots)
    arena.all_reduce(group)
    for (name, c), h in zip(entries, head):
        n = h[0]
        if n == 0:
            continue
        if c.slots is None:  # adopt the merged statistic of a layer owned by another rank
            c._slots = arena.view(name).clone()
            c._shape = tuple(int(d) for d in h[3:3 + h[2]])
            c._dtype = _CODE_DTYPES.get(h[1], torch.float32)
        else:
            c.slots.copy_(arena.view(name))
    return len(arena)


def sync_headroom_amax(model, group=None) -> int:
    """MAX-merge, across the ranks of ``group``, the ``_amax`` of every enabled quantizer whose calibrator is an
    ``NVFP4ActHeadroomCalibrator`` -- after the amaxes are loaded, since a headroom amax is a percentile rule, not a
    running max that ``sync_calibrator_amax`` could merge slot by slot.  One all-reduce over a flat fp32 buffer
    (``named_modules`` order, zeros where a rank holds no amax): the result is the largest per-rank scale
    (quantization/model_calib.py:606-609).  A quantizer that holds no amax here adopts a positive merged one.  Returns
    the number of quantizers merged."""
    from .calib import NVFP4ActHeadroomCalibrator
    from .nn import TensorQuantizer

    qs = [q for _, q in model.named_modules()
          if isinstance(q, TensorQuantizer) and not q._disabled and isinstance(q._calibrator, NVFP4ActHeadroomCalibrator)]
    if not qs:
        return 0
    device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" \
        else torch.device("cpu")
    zero = torch.zeros((), dtype=torch.float32, device=device)
    buf = torch.stack([q._amax.detach().reshape(()).to(device, torch.float32) if hasattr(q, "_amax") else zero
                       for q in qs])
    dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=group)
    for q, v in zip(qs, buf):
        if hasattr(q, "_amax"):
            q._amax.copy_(v.reshape(q._amax.shape))
        elif float(v) > 0:
            q.amax = v.clone()
    return len(qs)


__all__ = ["AmaxArena", "is_initialized", "shard_layers", "sync_calibrator_amax", "sync_headroom_amax"]
