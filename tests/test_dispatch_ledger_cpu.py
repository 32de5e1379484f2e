"""The launch-variant ledger (tests/_dispatch_ledger.py) names every ``__global__`` kernel in the CUDA sources and
nothing else, so a new kernel cannot ship without saying which test holds each of its instantiations to the oracle."""

import os
import re

import pytest

import _dispatch_ledger as ledger

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "model_optimizer_b200", "csrc")

_GLOBAL = re.compile(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\s*\((?:[^()]|\([^()]*\))*\)\s*)?(?:void\s+)?"
                     r"(\w+)\s*\(")


def kernels_in(text: str) -> set:
    text = re.sub(r"//[^\n]*", "", text)
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(_GLOBAL.findall(text))


def source_kernels() -> dict:
    found = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, f)) as fh:
                for k in kernels_in(fh.read()):
                    found.setdefault(k, f)
    return found


def test_scanner_finds_kernel_definitions():
    src = """
    template <typename Tag, int VB>
    __global__ void __launch_bounds__(kThreads, (N > 1) ? 2 : 1)
        a_kernel(const void *x) {}
    __global__ void b_kernel(int n) {}
    // __global__ void commented_out(int n) {}
    __global__ void
    c_kernel(int n);
    """
    assert kernels_in(src) == {"a_kernel", "b_kernel", "c_kernel"}


def test_every_kernel_has_a_ledger_entry_and_every_entry_a_kernel():
    src = source_kernels()
    assert len(src) > 50, sorted(src)
    missing = sorted(set(src) - set(ledger.LEDGER))
    stale = sorted(set(ledger.LEDGER) - set(src))
    assert not missing, f"__global__ kernels without a ledger entry in tests/_dispatch_ledger.py: {missing}"
    assert not stale, f"ledger entries naming kernels that no longer exist: {stale}"
    for k, e in ledger.LEDGER.items():
        assert e["file"] == src[k], (k, e["file"], src[k])


@pytest.mark.parametrize("kernel", sorted(ledger.LEDGER))
def test_ledger_entry_is_well_formed(kernel):
    e = ledger.LEDGER[kernel]
    header = open(os.path.join(ROOT, "include", "b200quant.h")).read()
    assert e["entry"] and e["variants"], kernel
    for fn in e["entry"]:
        assert re.search(rf"\b{fn}\s*\(", header), (kernel, fn)
    names = [v[0] for v in e["variants"]]
    assert len(set(names)) == len(names), (kernel, "duplicate variants")
    for name, cond, test in e["variants"]:
        assert name == f"b200q::{kernel}" or name.startswith(f"b200q::{kernel}<"), (kernel, name)
        assert cond, (kernel, name)
        assert os.path.exists(os.path.join(ROOT, test)), (kernel, name, test)


def test_canonical_names_match_both_demangler_spellings():
    rx = ledger.variant_regex("b200q::nvfp4_pack_kernel<{T}, 16, true, 1>")
    for raw in ("void b200q::nvfp4_pack_kernel<b200q::F16Tag, 16, true, 1>(unsigned char const*, unsigned long, int)",
                "void b200q::nvfp4_pack_kernel<b200q::F16Tag, (int)16, (bool)1, (int)1>(const unsigned char *, int)"):
        assert rx.match(ledger.canonical(raw)), ledger.canonical(raw)
    assert not rx.match(ledger.canonical("void b200q::nvfp4_pack_kernel<b200q::F16Tag, 32, true, 1>(int)"))
    assert not ledger.variant_regex("b200q::amax_rows_kernel<{T}, 32, 2>").match(
        ledger.canonical("void b200q::amax_rows_kernel<b200q::BF16Tag, 32, 32>(int)"))
    assert ledger.variant_regex("b200q::mx_fq_kernel<{T}, 2, *>").match(
        ledger.canonical("void b200q::mx_fq_kernel<b200q::BF16Tag, (int)2, (int)6>(const unsigned char *)"))
    assert ledger.canonical("b200q::hist_plan_kernel(float const*, int)") == "b200q::hist_plan_kernel"
