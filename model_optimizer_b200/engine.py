"""Layer-sharded PTQ hot-path engine.

Drives the three numeric hot paths for a whole decoder-only model whose linears are described by a
``ModelPlan`` (shapes only -- the GEMMs / attention are not part of this engine):

  collect   : every input quantizer folds |x| max of its activation batch into ONE flat fp32 arena
              (``distributed.AmaxArena``), one fused kernel per quantizer;
  finish    : the arena is all-reduced once (MAX, NCCL over NVLink) and exported to the quantizers'
              ``_amax`` buffers (views into one flat arena in the activation dtype) with one kernel;
  fake quant: every input quantizer runs its fused fake-quant forward (NVFP4 / FP8 / INT8);
  weights   : per-tensor amax + quant-and-pack of every owned weight.

``calib="nvfp4_act_headroom"`` (NVFP4, one GPU) calibrates with the NVFP4 activation-headroom rule instead of max:
collect adds every activation's per-block log2 histogram and running max to one ``[n_quantizers, 512]`` int64 table
(one grouped launch), and ``finish`` turns each histogram into an fp32 amax on the host, once per job.

Decoder layers are sharded contiguously over ranks (``distributed.shard_layers``); the statistics of
different layers are independent, so the only collective is the arena all-reduce -- ONE per calibration job
(``allreduce_every`` batches, 64 for 512 samples x batch 8), issued on a communication stream.  The ranks form a
pipeline: every step a rank receives the hidden state ``[tokens, hidden]`` of the NEXT micro-batch from rank - 1
(it is the input of its first layer's q/k/v quantizers) and hands its own last hidden state to rank + 1 on the
communication stream: a copy kernel that stores straight into the next rank's inbox (symmetric memory over NVLink /
NVSwitch, two device-side barriers around it; NCCL send / recv as the fallback), double-buffered by step parity and one
step ahead of its consumer so that the transfer overlaps the kernels of the following step.  The per-batch launch sequences are captured into CUDA graphs (static
activation buffers, one graph set per parity).
"""

from __future__ import annotations

import os

from dataclasses import dataclass

import torch

from . import ops
from .calib import MaxCalibrator, NVFP4ActHeadroomCalibrator
from .config import NVFP4ActHeadroomCalibConfig, QuantizerAttributeConfig
from .distributed import AmaxArena, shard_layers
from .nn import TensorQuantizer


@dataclass(frozen=True)
class ModelPlan:
    name: str
    hidden: int
    intermediate: int
    n_layers: int
    kv_dim: int

    def linears(self):
        """(name, in_features, out_features) of the 7 quantized linears of one decoder layer."""
        h, i, kv = self.hidden, self.intermediate, self.kv_dim
        return [("q_proj", h, h), ("k_proj", h, kv), ("v_proj", h, kv), ("o_proj", h, h),
                ("gate_proj", h, i), ("up_proj", h, i), ("down_proj", i, h)]

    def act_elems_per_token(self) -> int:
        return sum(cin for _, cin, _ in self.linears())

    def weight_elems_per_layer(self) -> int:
        return sum(cin * cout for _, cin, cout in self.linears())


LLAMA3_8B = ModelPlan("llama-3-8b", 4096, 14336, 32, 1024)
LLAMA3_70B = ModelPlan("llama-3-70b", 8192, 28672, 80, 1024)
TINY = ModelPlan("tiny", 256, 512, 4, 64)
PLANS = {p.name: p for p in (LLAMA3_8B, LLAMA3_70B, TINY)}

_FORMATS = {
    "nvfp4": {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "dynamic", "scale_bits": (4, 3)}},
    "fp8": {"num_bits": (4, 3), "axis": None},
    "int8": {"num_bits": 8, "axis": None},
}


class ShardedPTQEngine:
    """One rank's share of the model's input quantizers (+ weights), bound to a global amax arena."""

    def __init__(self, plan: ModelPlan, tokens: int, qformat: str = "nvfp4", dtype=torch.bfloat16,
                 device="cuda", rank: int = 0, world_size: int = 1, group=None, allreduce_every: int = 64,
                 handoff: bool = True, dedupe_shared_inputs: bool = False, grouped: bool = True,
                 calib: str = "max", headroom: dict | None = None):
        """``calib``: ``"max"`` or ``"nvfp4_act_headroom"`` (NVFP4 and ``world_size == 1`` only); ``headroom``: the
        ``anchor_percentile`` / ``upper_percentile`` / ``rho`` of the latter (``NVFP4ActHeadroomCalibConfig``)."""
        if calib not in ("max", "nvfp4_act_headroom"):
            raise ValueError(f"calib must be 'max' or 'nvfp4_act_headroom', got {calib!r}")
        if calib == "nvfp4_act_headroom":
            if qformat != "nvfp4":
                raise ValueError("calib='nvfp4_act_headroom' calibrates NVFP4 input quantizers only")
            if world_size > 1:
                raise NotImplementedError("calib='nvfp4_act_headroom' runs on one GPU; a multi-GPU headroom engine "
                                          "is not implemented")
        elif headroom is not None:
            raise ValueError("headroom options need calib='nvfp4_act_headroom'")
        self.calib = calib
        self.plan, self.tokens, self.qformat, self.dtype = plan, tokens, qformat, dtype
        self.device = torch.device(device)
        self.rank, self.world_size, self.group = rank, world_size, group
        self.layers = list(shard_layers(plan.n_layers, world_size, rank))
        self.arena = AmaxArena(self.device)
        for layer in range(plan.n_layers):          # same layout on every rank
            for name, _, _ in plan.linears():
                self.arena.register(f"layers.{layer}.{name}.input_quantizer")
        self.arena.freeze()
        # _amax buffers of all quantizers live in one flat arena of the activation dtype
        self.amax_arena = torch.zeros(len(self.arena), dtype=dtype, device=self.device)
        self.quantizers: list[tuple[str, TensorQuantizer, int]] = []
        cfg = QuantizerAttributeConfig(**_FORMATS[qformat])
        idx = {n: i for i, n in enumerate(self.arena.names())}
        for layer in self.layers:
            for name, cin, _ in plan.linears():
                qn = f"layers.{layer}.{name}.input_quantizer"
                q = TensorQuantizer(cfg)
                cal = q._calibrator
                assert isinstance(cal, MaxCalibrator)
                cal._slots = self.arena.view(qn)      # collect kernels write straight into the arena
                cal._shape, cal._dtype = (), dtype
                q._amax = self.amax_arena[idx[qn]:idx[qn] + 1].view(())   # view: export fills it
                self.quantizers.append((qn, q, cin))
        self.hist = self.running_max = None
        if calib == "nvfp4_act_headroom":
            # every quantizer's histogram and running max are rows of one table (the grouped launch fills them all);
            # its fp32 amax is its arena slot, which finish() writes and the fake quant reads as it is (no export)
            hc = NVFP4ActHeadroomCalibConfig(**(headroom or {}))
            n = len(self.quantizers)
            self.hist = torch.zeros(n, 512, dtype=torch.int64, device=self.device)
            self.running_max = torch.zeros(n, dtype=torch.float32, device=self.device)
            for i, (qn, q, _) in enumerate(self.quantizers):
                cal = NVFP4ActHeadroomCalibrator(anchor_percentile=hc.anchor_percentile,
                                                 upper_percentile=hc.upper_percentile, rho=hc.rho)
                cal._hist, cal._running_max, cal._dtype = self.hist[i], self.running_max[i:i + 1], dtype
                q._calibrator = cal
                q._amax = self.arena.view(qn).view(())
        self._tables = {}
        self._graphs = {}
        self._graph_sets = []
        self.allreduce_every = max(1, int(allreduce_every))
        self.handoff = bool(handoff) and world_size > 1
        self.dedupe_shared_inputs = bool(dedupe_shared_inputs)
        # grouped = ONE multi-tensor launch for the collect of all owned quantizers and ONE for their NVFP4 fake
        # quant (pointer-array kernels) instead of one launch per quantizer
        self.grouped = bool(grouped) and qformat == "nvfp4"
        # grouped graph steps: number of quantizers whose fake quant the fix-up redid since reset() (int32 device
        # scalar); in a steady state, where no batch sets a new running max, it stops growing
        self.redo_count = torch.zeros(1, dtype=torch.int32, device=self.device) if self.grouped else None
        self._fixup_bytes = 0
        self._step = 0
        self.comm_log = {"allreduce_calls": 0, "p2p_calls": 0, "p2p_bytes": 0}
        # layer sharding: a rank's fake quant only needs the amax of its OWN layers, which is complete
        # locally; the all-reduce only replicates the full arena on every rank (export / checkpoint).  So
        # it runs on a side stream over a staging copy and overlaps the fake-quant phase.
        self.global_arena = torch.zeros_like(self.arena.freeze()) if world_size > 1 else self.arena.freeze()
        self._comm_stream = torch.cuda.Stream(self.device) if world_size > 1 and self.device.type == "cuda" else None
        self._ev_collected = torch.cuda.Event() if self._comm_stream is not None else None
        if self.handoff:
            h = (tokens, plan.hidden)
            # parity-double-buffered hand-off buffers: hand_in[p] feeds the first owned layer's q/k/v quantizers in
            # steps of parity p (ranks > 0), hand_out[p] is what this rank's last layer produced in such a step
            self.hand_out = [torch.zeros(h, dtype=dtype, device=self.device) for _ in range(2)] \
                if rank < world_size - 1 else None
            self._ev_step_done = [torch.cuda.Event() for _ in range(2)]
            self._ev_comm = [torch.cuda.Event() for _ in range(2)]
            # The inbox (hand_in) lives in SYMMETRIC memory when it can: the hand-off is then a plain copy kernel
            # that stores into the next rank's inbox over NVLink / NVSwitch peer memory (full link bandwidth at
            # any world size) bracketed by two device-side barriers, instead of an NCCL send / recv pair (whose
            # point-to-point channel count shrinks with the communicator size: 415 GB/s at N = 2 but 81 GB/s at
            # N = 8).  Setup failure -> the NCCL path below.
            self._symm = None
            self._peer_in = None
            self.handoff_transport = "nccl send/recv"
            inbox = None
            if os.environ.get("B200Q_HANDOFF", "symm") != "nccl" and self.device.type == "cuda":
                try:
                    import torch.distributed as dist
                    import torch.distributed._symmetric_memory as symm_mem

                    n = tokens * plan.hidden
                    grp = group if group is not None else dist.group.WORLD
                    inbox = symm_mem.empty(2 * n, dtype=dtype, device=self.device)
                    inbox.zero_()
                    self._symm = symm_mem.rendezvous(inbox, grp)
                    if rank < world_size - 1:
                        self._peer_in = [self._symm.get_buffer(rank + 1, (n,), dtype, q * n) for q in range(2)]
                    self.handoff_transport = "peer-memory copy (symmetric memory) + device barriers"
                except Exception as e:  # noqa: BLE001
                    self._symm, self._peer_in, inbox = None, None, None
                    self.handoff_fallback_reason = repr(e)[:200]
            if self.device.type == "cuda":                   # every rank must have taken the same path
                import torch.distributed as dist

                flag = torch.tensor([1 if self._symm is not None else 0], device=self.device, dtype=torch.int32)
                dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
                if int(flag.item()) == 0 and self._symm is not None:
                    self._symm, self._peer_in, inbox = None, None, None
                    self.handoff_transport = "nccl send/recv"
                    self.handoff_fallback_reason = "symmetric memory unavailable on another rank"
            if rank > 0:
                if inbox is not None:
                    n = tokens * plan.hidden
                    self.hand_in = [inbox[q * n:(q + 1) * n].view(h) for q in range(2)]
                else:
                    self.hand_in = [torch.zeros(h, dtype=dtype, device=self.device) for _ in range(2)]
            else:
                self.hand_in = None
            self._inbox = inbox

    # ---- buffers -------------------------------------------------------------------------------------
    def alloc_activations(self, seed: int = 0, distinct: bool = True):
        """Synthetic bf16 activations [tokens, Cin], one per owned quantizer (distinct buffers: no L2
        reuse between quantizers that would share an input in a real model)."""
        g = torch.Generator(device=self.device).manual_seed(seed + 1000 * self.rank)
        acts = []
        cache = {}
        for _, _, cin in self.quantizers:
            if not distinct and cin in cache:
                acts.append(cache[cin])
                continue
            x = torch.randn(self.tokens, cin, device=self.device, generator=g, dtype=torch.float32).to(self.dtype)
            cache[cin] = x
            acts.append(x)
        return acts

    def acts_for_parity(self, acts, p: int):
        """The activation list of steps with parity p: on ranks > 0 the inputs of the first owned layer's q/k/v
        quantizers are the hand-off buffer received for that step."""
        if not self.handoff or self.hand_in is None:
            return acts
        acts = list(acts)
        for i, (qn, _, cin) in enumerate(self.quantizers[:3]):
            assert cin == self.plan.hidden, qn
            acts[i] = self.hand_in[p]
        return acts

    def alloc_outputs(self, n_ring: int = 4):
        cmax = max(cin for _, _, cin in self.quantizers)
        return [torch.empty(self.tokens * cmax, dtype=self.dtype, device=self.device) for _ in range(n_ring)]

    # ---- the hot path ----------------------------------------------------------------------------------
    def collect(self, acts):
        """Calibration collect of one batch: one fused |x|-max kernel per quantizer.  Headroom mode: one grouped
        histogram launch over every activation (``grouped``), else one calibrator collect per quantizer."""
        if self.hist is not None and self.grouped:
            ops.nvfp4_block_log2_hist_multi_(self.hist, self.running_max, self._cached_table(acts))
            return
        for (_, q, _), x in zip(self.quantizers, acts):
            q._calibrator.collect(x)

    def _cached_table(self, acts, ys=None):
        """The descriptor table of these (static) buffers, built on first use -- outside any graph capture, since the
        build copies the table to the device.  Slot i = quantizer i."""
        key = (tuple(x.data_ptr() for x in acts), None if ys is None else tuple(y.data_ptr() for y in ys))
        t = self._tables.get(key)
        if t is None:
            if ys is not None:
                spans = sorted((y.data_ptr(), y.data_ptr() + y.numel() * y.element_size()) for y in ys)
                if any(b[0] < a[1] for a, b in zip(spans, spans[1:])):
                    raise ValueError("the grouped headroom fake quant needs non-overlapping outputs "
                                     "(alloc_outputs(n_ring=len(engine.quantizers)))")
            t = ops.TensorTable(acts, list(range(len(acts))), ys, "block16")
            self._tables[key] = t
        return t

    def _table(self, acts, outs, parity):
        """Descriptor table of a parity's static buffers for the fused collect + fake quant: every owned quantizer's
        activation with its arena slot and its fake-quant destination (a ring of ``outs``; the hand-off buffer for the
        last o_proj).  Raises if an output overlaps an activation or two outputs overlap other than as prefixes of one
        buffer."""
        idx = {n: i for i, n in enumerate(self.arena.names())}
        slots = [idx[qn] for qn, _, _ in self.quantizers]
        n = len(outs)
        last_hidden = len(self.quantizers) - 4 if (self.handoff and self.hand_out is not None) else -1
        ys = [self.hand_out[parity] if i == last_hidden else outs[i % n][: x.numel()].view_as(x)
              for i, x in enumerate(acts)]
        return ops.TensorTable(acts, slots, ys, "block16", fused=True)

    def _capture_set(self, acts, outs, parity, side):
        g_collect, g_export, g_fq = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        if self.hist is not None:
            # headroom: the amax is not a running max, so the speculative fused pass cannot be fixed up; the step is
            # collect, then fake quant with the amaxes of the last finish()
            with torch.cuda.graph(g_collect, stream=side):
                self.collect(acts)
            with torch.cuda.graph(g_fq, stream=side):
                self.fake_quant(acts, outs, parity)
            return {"collect": g_collect, "fake_quant": g_fq}
        if self.grouped:
            # ONE read of every activation per step: the fused pass fake-quantizes with the amax exported by the
            # previous step while it collects; the fix-up redoes the (rare) entries whose exported amax changes.
            # Graph keys: "fake_quant" is the fused pass (the NVFP4 grid, 4 B per element), "collect" the fix-up.
            t = self._table(acts, outs, parity)
            self._fixup_bytes = t.fixup_bytes
            arena = self.arena.freeze()

            def fused():
                ops.collect_fake_quant_nvfp4_multi(t, arena, self.amax_arena)

            def fixup():
                ops.fake_quant_nvfp4_multi_fixup(t, arena, self.amax_arena, self.redo_count)

            with torch.cuda.stream(side):
                fused()
                fixup()
            torch.cuda.synchronize(self.device)
            self.reset()
            with torch.cuda.graph(g_fq, stream=side):
                fused()
            with torch.cuda.graph(g_collect, stream=side):
                fixup()
            with torch.cuda.graph(g_export, stream=side):
                self.export_amax()
            return {"collect": g_collect, "export": g_export, "fake_quant": g_fq, "tables": (t,)}
        with torch.cuda.graph(g_collect, stream=side):
            self.collect(acts)
        with torch.cuda.graph(g_export, stream=side):
            self.export_amax()
        with torch.cuda.graph(g_fq, stream=side):
            self.fake_quant(acts, outs, parity)
        return {"collect": g_collect, "export": g_export, "fake_quant": g_fq}

    def finish(self):
        """One collective + one export kernel: arena (fp32) -> all quantizers' _amax (input dtype).  Headroom mode:
        the histogram table comes to the host in one copy, every quantizer's amax is computed there, and the fp32
        amaxes go to the arena slots the fake quant reads."""
        if self.hist is not None:
            counts, rmax = self.hist.cpu(), self.running_max.cpu().tolist()
            amax = [q._calibrator.amax_from_host(counts[i], rmax[i]) for i, (_, q, _) in enumerate(self.quantizers)]
            self.arena.freeze().copy_(torch.tensor([0.0 if a is None else a for a in amax], dtype=torch.float32))
            return
        if self.world_size > 1:
            self.arena.all_reduce(self.group)
        self.export_amax()

    def export_amax(self):
        _lib_call_export(self.arena.freeze(), self.amax_arena)

    def fake_quant(self, acts, outs, parity: int = 0):
        """Fake-quant forward of one batch with the calibrated amax: one fused kernel per quantizer.  With the
        hand-off enabled the o_proj input of the LAST owned layer ([tokens, hidden]) lands in ``hand_out[parity]``:
        the buffer this rank sends on (a stand-in for the layer output the GEMMs would produce)."""
        n = len(outs)
        res = []
        if self.hist is not None and self.grouped:
            ys = [outs[i % n][: x.numel()].view_as(x) for i, x in enumerate(acts)]
            ops.fake_quant_nvfp4_multi(self._cached_table(acts, ys), self.arena.freeze())
            return ys
        last_hidden = len(self.quantizers) - 4 if (self.handoff and self.hand_out is not None) else -1
        for i, ((_, q, _), x) in enumerate(zip(self.quantizers, acts)):
            out = self.hand_out[parity] if i == last_hidden else outs[i % n][: x.numel()].view_as(x)
            if self.qformat == "nvfp4":
                ops.fake_quant_nvfp4(x, q._amax, out=out)
            elif self.qformat == "fp8":
                ops.fake_quant_fp8(x, q._amax, out=out)
            else:
                ops.fake_quant_int(x, q._amax, 8, False, False, out=out)
            res.append(out)
        return res

    def reset(self):
        self.arena.freeze().zero_()
        self.amax_arena.zero_()
        if self.redo_count is not None:
            self.redo_count.zero_()
        if self.hist is not None:
            self.hist.zero_()
            self.running_max.zero_()

    # ---- CUDA graphs -----------------------------------------------------------------------------------
    def capture(self, acts, outs):
        """Capture the collect and fake-quant launch sequences of one batch (static buffers); with the hand-off,
        one graph set per step parity."""
        torch.cuda.synchronize(self.device)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            self.collect(acts)       # warm-up outside capture (module / kernel loading, descriptor tables)
            if self.hist is None:
                self.export_amax()
            self.fake_quant(acts, outs)
        torch.cuda.synchronize(self.device)
        self.reset()
        self._graph_sets = [self._capture_set(self.acts_for_parity(acts, p), outs, p, side)
                            for p in range(2 if self.handoff else 1)]
        self._graphs = self._graph_sets[0]
        self.reset()
        self._step = 0
        return self._graphs

    def all_reduce_async(self):
        """THE collective, off the critical path: copy the local arena to the staging buffer and
        all-reduce(MAX) it on the communication stream; ``wait_all_reduce`` joins it."""
        import torch.distributed as dist

        main = torch.cuda.current_stream(self.device)
        self._ev_collected.record(main)
        with torch.cuda.stream(self._comm_stream):
            self._comm_stream.wait_event(self._ev_collected)
            self.global_arena.copy_(self.arena.freeze(), non_blocking=True)
            dist.all_reduce(self.global_arena, op=dist.ReduceOp.MAX, group=self.group)

    def wait_all_reduce(self):
        torch.cuda.current_stream(self.device).wait_stream(self._comm_stream)

    def _exchange(self, q: int):
        """Communication stream: move ``hand_out[q]`` (written by the last parity-q step) into rank + 1's ``hand_in[q]``
        and receive the input of the NEXT parity-q step from rank - 1 (peer-memory copy between two device barriers, or
        one NCCL send / recv group on the fallback path).  It is issued
        at the START of the following step, so the transfer runs under that step's kernels (which touch the other
        parity's buffers): a pipeline with one step of slack, as a layer-sharded forward has between micro-batches."""
        import torch.distributed as dist

        if self._symm is not None:
            nbytes = 0
            with torch.cuda.stream(self._comm_stream):
                self._comm_stream.wait_event(self._ev_step_done[q])
                self._symm.barrier(channel=0)               # every rank finished the step that last read inbox[q]
                if self._peer_in is not None:
                    self._peer_in[q].copy_(self.hand_out[q].reshape(-1))   # stores into rank + 1's inbox over NVLink
                    nbytes = self.hand_out[q].numel() * self.hand_out[q].element_size()
                self._symm.barrier(channel=1)               # every inbox of this round is complete
                self._ev_comm[q].record(self._comm_stream)
            self.comm_log["p2p_calls"] += 1 if nbytes else 0
            self.comm_log["p2p_bytes"] += nbytes
            return
        with torch.cuda.stream(self._comm_stream):
            self._comm_stream.wait_event(self._ev_step_done[q])
            reqs = []
            if self.hand_out is not None:
                reqs.append(dist.P2POp(dist.isend, self.hand_out[q], self.rank + 1, self.group))
            if self.hand_in is not None:
                reqs.append(dist.P2POp(dist.irecv, self.hand_in[q], self.rank - 1, self.group))
            for w in dist.batch_isend_irecv(reqs):
                w.wait()                                  # stream-level wait on the communication stream
            self._ev_comm[q].record(self._comm_stream)
        self.comm_log["p2p_calls"] += len(reqs)
        self.comm_log["p2p_bytes"] += sum(r.tensor.numel() * r.tensor.element_size() for r in reqs)

    def step_graph(self):
        """One batch as graph replays: collect -> export -> fake quant, or with ``grouped`` the fused collect + fake
        quant -> fix-up -> export (same results).  Communication stream, overlapped: the
        hidden-state hand-off of the PREVIOUS step's output (every step) and the arena all-reduce (once per
        ``allreduce_every`` batches)."""
        p = self._step & 1 if self.handoff else 0
        g = self._graph_sets[p] if self._graph_sets else self._graphs
        main = torch.cuda.current_stream(self.device)
        self._flushed_at = None
        if self.handoff and self._step >= 1:
            if self._step >= 2:
                # the exchange issued one step ago (parity p) delivered this step's input and released hand_out[p]
                main.wait_event(self._ev_comm[p])
            self._exchange(1 - p)                         # previous step's output travels under this step's kernels
        if self.hist is not None:
            g["collect"].replay()
            g["fake_quant"].replay()
        elif self.grouped:
            g["fake_quant"].replay()
            g["collect"].replay()
            g["export"].replay()
        else:
            g["collect"].replay()
            g["export"].replay()
            g["fake_quant"].replay()
        if self.handoff:
            self._ev_step_done[p].record(main)
        self._step += 1
        if self.world_size > 1 and self._step % self.allreduce_every == 0:
            self.all_reduce_async()
            self.comm_log["allreduce_calls"] += 1

    def join_comm(self):
        """Join the communication stream (end of a calibration job / of a timed region); the last step's output is
        handed off first so that a job of K steps moves K hidden states."""
        if self._comm_stream is not None:
            if self.handoff and self._step >= 1 and not getattr(self, "_flushed_at", None) == self._step:
                self._exchange((self._step - 1) & 1)
                self._flushed_at = self._step
            torch.cuda.current_stream(self.device).wait_stream(self._comm_stream)

    def launches_per_step(self) -> int:
        if self.hist is not None:
            return 2 if self.grouped else 2 * len(self.quantizers)
        return 3 if self.grouped else 2 * len(self.quantizers) + 1

    def act_bytes_per_step(self) -> tuple[int, int]:
        """(collect bytes, fake-quant bytes) of algorithmic HBM traffic for one batch on this rank.  ``grouped``: the
        collect rides on the fake-quant read, and the first item is the fix-up's traffic when no exported amax changes
        (the live blocks of the pre-flagged output tiles it rewrites, ``ops.output_tiles``; known once captured)."""
        elems = sum(self.tokens * cin for _, _, cin in self.quantizers)
        es = torch.empty((), dtype=self.dtype).element_size()
        return self._fixup_bytes if self.grouped and self.hist is None else elems * es, 2 * elems * es

    # ---- weights -----------------------------------------------------------------------------------------
    def weight_pass(self, weights):
        """Per-tensor amax + NVFP4 (or FP8) quant-and-pack of every owned weight; returns packed tensors."""
        out = []
        for w in weights:
            slot = torch.zeros(1, dtype=torch.float32, device=w.device)
            ops.amax_per_tensor_(slot, w)
            if self.qformat == "nvfp4":
                out.append(ops.pack_nvfp4(w, slot))
            else:
                scale = slot / torch.tensor(448.0, device=w.device)
                out.append((ops.pack_fp8(w, scale), scale))
        return out


def _lib_call_export(slots: torch.Tensor, dst: torch.Tensor):
    from ._lib import call
    from .ops import _DT, _stream

    call("b200q_amax_export", slots.data_ptr(), slots.numel(), dst.data_ptr(), _DT[dst.dtype], _stream(slots))


__all__ = ["ModelPlan", "PLANS", "LLAMA3_8B", "LLAMA3_70B", "TINY", "ShardedPTQEngine"]
