"""Inputs of the exhaustive value sweep (``tests/test_gpu_value_sweep.py``) and the host-side branch conditions of the
kernels it reaches (checked by ``tests/test_value_sweep_cpu.py``, so that an edit of the grid cannot quietly stop
reaching a branch).

The element domain is every bit pattern of a 16-bit type and, for fp32, every biased exponent with edge mantissas plus
the values on and next to each rounding boundary of the format at the scale in use.  The scale grid ``S`` spans the
whole fp32 range and straddles every window edge of the exact division (``ExactDiv`` in ``csrc/common.cuh``) and the
other scale thresholds of the quantizers."""

from __future__ import annotations

import numpy as np

from oracle import oracle_np as o

F32 = np.float32
FLT_MAX = F32(np.finfo(np.float32).max)
DENORM_MIN = F32(2.0 ** -149)

# ExactDiv::div's operand window (2^-60, 2^60), the block window [kBlockMin, kBlockMax] = [2^-40, 2^60] and the NVFP4
# pack's kMaxDenom (1.0 for fp32, 2^16 for bf16)
EDGES = (2.0 ** -60, 2.0 ** -40, 1.0, 2.0 ** 16, 2.0 ** 60)
# amax <= 2^-24 zeroes the INT / FP8 fake quant; a dynamic NVFP4 block scale below 1e-5 becomes 1
THRESHOLDS = (2.0 ** -24, 1e-5)
K_BLOCK_MIN, K_BLOCK_MAX = 2.0 ** -40, 2.0 ** 60
K_MAX_DENOM = {"bf16": 2.0 ** 16, "f16": 2.0 ** 60, "f32": 1.0}
DTYPES = ("bf16", "f16", "f32")


def around(v):
    """v and its two fp32 neighbours."""
    v = F32(v)
    return [np.nextafter(v, F32(-np.inf)), v, np.nextafter(v, F32(np.inf))]


def scale_grid(stride: int = 6) -> np.ndarray:
    """The scale grid S (sorted fp32): powers of two 2^-133 .. 2^127 every ``stride`` binades, every edge and threshold
    with its fp32 neighbours, a few non-power-of-two mantissas, and 0, the smallest denormal and FLT_MAX."""
    s = {F32(2.0 ** e) for e in range(-133, 128, stride)} | {F32(2.0 ** 127)}
    for edge in EDGES + THRESHOLDS:
        s.update(around(edge))
    for m in (1.5, 1.75, 7.0 / 6.0):
        for e in (-126, -60, -20, 0, 20, 60, 120):
            s.add(F32(m * 2.0 ** e))
    s.update((F32(0.0), DENORM_MIN, FLT_MAX))
    return np.array(sorted(s), dtype=F32)


def coarse(s: np.ndarray, every: int = 4) -> np.ndarray:
    """A subset of S for the launches that take one scale each: every ``every``-th point plus all edge points."""
    keep = np.zeros(s.size, dtype=bool)
    keep[::every] = True
    for edge in EDGES + THRESHOLDS:
        keep |= np.isin(s, np.array(around(edge), dtype=F32))
    keep[-1] = keep[0] = True
    return s[keep]


# ------------------------------------------------------------------------------------------------
# element domain
# ------------------------------------------------------------------------------------------------
def patterns16() -> np.ndarray:
    """All 65536 bit patterns of a 16-bit type, as uint16."""
    return np.arange(65536, dtype=np.uint32).astype(np.uint16)


def values16(dt: str) -> np.ndarray:
    """fp32 values of all 65536 patterns of ``dt`` ("bf16" / "f16"), in pattern order."""
    p = patterns16()
    if dt == "bf16":
        return (p.astype(np.uint32) << 16).view(F32)
    return p.view(np.float16).astype(F32)


FP32_MANTISSAS = (0, 1, 2, 0x3FFFFF, 0x400000, 0x400001, 0x7FFFFE, 0x7FFFFF)


def fp32_structured(seed: int = 0) -> np.ndarray:
    """Every biased exponent 0..255 x the edge mantissas and a few seeded ones x both signs (6144 values)."""
    rng = np.random.default_rng(seed)
    mants = np.array(FP32_MANTISSAS + tuple(int(m) for m in rng.integers(3, 0x7FFFFD, 4)), dtype=np.uint32)
    e = np.arange(256, dtype=np.uint32)
    bits = ((e[:, None] << 23) | mants[None, :]).reshape(-1)
    return np.concatenate([bits, bits | np.uint32(0x80000000)]).view(F32)


def _midpoints(v):
    v = np.asarray(v, dtype=np.float64)
    return (v[1:] + v[:-1]) / 2


def e4m3_positive():
    return np.unique(o.e4m3_from_bits(np.arange(0x7F, dtype=np.uint8)))


# rounding boundaries t of each format, in units of the quantization step (the value x / scale takes there)
E2M1_T = (0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, 6.0)
E4M3_T = tuple(_midpoints(e4m3_positive())) + (448.0, 464.0)
NF4_T = tuple(_midpoints(o.NF4_LUT)) + (1.0,)


def int_t(bound: int):
    return tuple(k + 0.5 for k in range(bound + 1))


def boundary_values(unit, ts) -> np.ndarray:
    """fl(unit * t) and its two fp32 neighbours for every boundary t, both signs."""
    with np.errstate(over="ignore", under="ignore"):
        v = np.array([F32(F32(unit) * F32(t)) for t in ts], dtype=F32)
        v = np.concatenate([np.nextafter(v, F32(-np.inf)), v, np.nextafter(v, F32(np.inf))])
    return np.concatenate([v, -v]).astype(F32)


def fp32_rows(units, ts, mult: int = 32) -> np.ndarray:
    """[len(units), L]: each row the structured fp32 set plus the boundary values of its own unit, zero padded to a
    multiple of ``mult``."""
    base = fp32_structured()
    rows = [np.concatenate([base, boundary_values(u, ts)]) for u in units]
    n = len(rows[0])
    n_pad = -(-n // mult) * mult
    out = np.zeros((len(rows), n_pad), dtype=F32)
    for i, r in enumerate(rows):
        out[i, :n] = r
    return out


def domain(dt: str) -> np.ndarray:
    """The element domain of ``dt`` without per-scale boundary values: all patterns, or the structured fp32 set."""
    return values16(dt) if dt != "f32" else fp32_structured()


def dtype_max(dt: str) -> F32:
    return {"bf16": F32(o.from_bf16_bits(np.uint16(0x7F7F))), "f16": F32(65504.0), "f32": FLT_MAX}[dt]


def round_up_to(v, dt):
    """The smallest value of ``dt`` >= v (v >= 0), or dt's largest finite value when v is above it."""
    v = F32(v)
    r = F32(o.round_to(np.array([v], dtype=F32), dt)[0])
    if r < v:
        r = F32(o.round_to(np.array([np.nextafter(v, F32(np.inf))], dtype=F32), dt)[0])
        if r < v:       # fp16's grid is coarser than one fp32 step
            r = F32(o.round_to(np.array([v * F32(1.001)], dtype=F32), dt)[0])
    return r if np.isfinite(r) else dtype_max(dt)


def setter_blocks(pool, setters, block: int) -> np.ndarray:
    """Blocks of ``block`` elements: element 0 of block k is ``setters[k % len(setters)]``, the others walk through
    ``pool`` in order (every pool value lands in one block); [n_blocks, block]."""
    pool = np.asarray(pool, dtype=F32)
    fill = block - 1
    n_blocks = -(-pool.size // fill)
    body = np.zeros(n_blocks * fill, dtype=F32)
    body[:pool.size] = pool
    out = np.empty((n_blocks, block), dtype=F32)
    out[:, 1:] = body.reshape(n_blocks, fill)
    s = np.asarray(setters, dtype=F32)
    out[:, 0] = s[np.arange(n_blocks) % s.size]
    return out


def nvfp4_dynamic_input(dt: str, g) -> np.ndarray:
    """Input of the dynamic NVFP4 sweep at global amax ``g``: blocks led by +-(dt's max) or +-(the smallest dt value
    >= g), whose block scale clamps at 448 * g / 2688 = g / 6 whenever g fits dt, then the domain in natural blocks;
    [-1, 16]."""
    m = dtype_max(dt)
    gs = round_up_to(g, dt)
    lead = setter_blocks(domain(dt), [m, gs, -m, -gs], 16)
    tail = domain(dt).reshape(-1, 16)
    return np.concatenate([lead, tail])


def mx_setters(dt: str, step: int = 3) -> np.ndarray:
    """Positive setter magnitudes of ``dt`` whose exponents cover its whole range (subnormals included)."""
    lo = {"bf16": -133, "f16": -24, "f32": -149}[dt]
    hi = {"bf16": 127, "f16": 15, "f32": 127}[dt]
    v = []
    for e in range(lo, hi + 1, step):
        for m in (1.0, 1.5, 1.99):
            v.append(F32(m * 2.0 ** e) if e > -149 or m == 1.0 else F32(2.0 ** e))
    v = o.round_to(np.array(v, dtype=F32), dt)
    v = v[np.isfinite(v) & (v > 0)]
    return np.unique(np.concatenate([v, [dtype_max(dt)]]).astype(F32))


def mx_input(dt: str, block: int, per_setter: int = 4) -> np.ndarray:
    """Input of the MX sweeps: for each setter, ``per_setter`` blocks led by it (alternating sign) and filled with
    finite domain values no larger than it (an evenly spread subset), then the whole domain in natural blocks;
    [-1, block]."""
    dom = domain(dt)
    fin = dom[np.isfinite(dom)]
    out = []
    for k, s in enumerate(mx_setters(dt)):
        small = fin[np.abs(fin) <= s]
        want = per_setter * (block - 1)
        idx = np.linspace(0, small.size - 1, want).round().astype(np.int64) if small.size else np.zeros(0, np.int64)
        pool = small[idx] if small.size else np.zeros(want, dtype=F32)
        out.append(setter_blocks(pool, [s, -s] if k % 2 else [-s, s], block))
    tail = np.zeros(-(-dom.size // block) * block, dtype=F32)
    tail[:dom.size] = dom
    out.append(tail.reshape(-1, block))
    return np.concatenate(out)


def wsf2_for_denom(target) -> F32:
    """A weights_scaling_factor_2 w with fl(448 * w) == target where one exists, else the closest w above."""
    w = F32(F32(target) / F32(448.0))
    for _ in range(8):
        d = F32(F32(448.0) * w)
        if d == F32(target):
            return w
        w = np.nextafter(w, F32(np.inf) if d < F32(target) else F32(-np.inf))
    return w


def pack_wsf2_grid() -> np.ndarray:
    """weights_scaling_factor_2 values of the NVFP4 pack sweep: the clamped block scale 448 * w then lands on every
    point of S in the window's neighbourhood, on each side of kBlockMin and of both kMaxDenom values."""
    s = coarse(scale_grid())
    s = s[s > 0]
    w = {wsf2_for_denom(v) for v in s}
    w.update(wsf2_for_denom(v) for e in (K_BLOCK_MIN, 1.0, 2.0 ** 16) for v in around(e))
    return np.array(sorted(w), dtype=F32)


# ------------------------------------------------------------------------------------------------
# the kernels' branch conditions, restated on the host
# ------------------------------------------------------------------------------------------------
def nvfp4_pack_denoms(x, global_amax=None, wsf2=None):
    """Per 16-element block of ``x`` [-1, 16]: (denom, finite block) of the dynamic NVFP4 pack (wsf2: given)."""
    x = np.asarray(x, dtype=F32)
    with np.errstate(all="ignore"):
        s2 = F32(wsf2) if wsf2 is not None else F32(F32(global_amax) / F32(6.0 * 448.0))
        bmax = np.max(np.abs(x), axis=-1)
        pbs = (bmax / F32(F32(6.0) * s2)).astype(F32)
        pbs = np.where(pbs == 0, F32(1.0), pbs)
        pbs = np.where(np.isnan(pbs), pbs, np.clip(pbs, F32(2.0 ** -9), F32(448.0))).astype(F32)
        bs_val, _ = o.e4m3fn_torch_cast(pbs)
        denom = (bs_val * s2).astype(F32)
    return denom, np.isfinite(bmax)


def nvfp4_pack_branches(x, dt, global_amax=None, wsf2=None):
    """Per block: (fast, overflow).  ``fast``: the window the pack's fast path takes (finite block, denom in
    [kBlockMin, kMaxDenom]); ``overflow``: a block in that window whose largest quotient |x| / denom overflows fp32."""
    denom, finite = nvfp4_pack_denoms(x, global_amax, wsf2)
    fast = finite & (denom >= F32(K_BLOCK_MIN)) & (denom <= F32(K_MAX_DENOM[dt]))
    with np.errstate(all="ignore"):
        q = (np.max(np.abs(np.asarray(x, dtype=F32)), axis=-1) / denom).astype(F32)
    return fast, fast & np.isinf(q)


def nvfp4_fq_block_ok(x, global_amax):
    """Per block of the dynamic NVFP4 fake quant: block_ok (finite block, scale in [kBlockMin, kBlockMax])."""
    x = np.asarray(x, dtype=F32)
    s = o.nvfp4_block_scale_dynamic(o.nan_skip_absmax(x, axis=-1), global_amax)
    return np.isfinite(np.max(np.abs(x), axis=-1)) & (s >= F32(K_BLOCK_MIN)) & (s <= F32(K_BLOCK_MAX))


def fp8_int8_pack_fast(x, s, int8: bool):
    """Per 16-element vector of the FP8 / INT8 pack (one scale per row of ``x`` [R, L]): the fast path's condition
    (s in ExactDiv's operand window, vmax <= 2^60 and, for FP8, vmax <= 448 * s)."""
    x = np.asarray(x, dtype=F32)
    s = np.asarray(s, dtype=F32).reshape(-1, 1)
    vmax = np.max(np.abs(x.reshape(x.shape[0], -1, 16)), axis=-1)
    ok = (s >= F32(2.0 ** -60)) & (s <= F32(2.0 ** 60)) & (s > 0)
    fast = ok & (vmax <= F32(2.0 ** 60))
    if not int8:
        with np.errstate(over="ignore"):
            fast &= vmax <= (F32(448.0) * s).astype(F32)
    return fast


def nf4_branches(x, s, dt):
    """Per 16-element block of the NF4 pack (``x`` [R, L], one scale per row): (fast, big) -- the scale window, and
    a fast block holding a quotient T(x / s) beyond +-4 (re-done in reference order)."""
    x = np.asarray(x, dtype=F32)
    s = np.asarray(s, dtype=F32).reshape(-1, 1)
    fast = (s >= F32(K_BLOCK_MIN)) & (s <= F32(K_BLOCK_MAX))
    with np.errstate(all="ignore"):
        v = o.round_to((x / s).astype(F32), dt)
    big = ~(np.abs(v.reshape(x.shape[0], -1, 16)) <= 4.0)
    big = big.any(axis=-1)
    return np.broadcast_to(fast, big.shape), fast & big
