"""Generate tests/golden/ref_export_formats*.npz: the reference's unified-HF export for every weight format the mirror
calibrates, including mixed-precision models.

Run from the repo root where the reference tree is available:  python tools/gen_export_formats_golden.py

Built like ``oracle/gen_golden.py::main_export``: the same tiny HF Llama and calibration data, ``mtq.quantize`` on CPU
with the same import shim, then the reference's own ``export_hf_checkpoint``.  The reference fake-quantizes dynamic
NVFP4 blocks only through CUDA code; for the AWQ searches (``NVFP4_AWQ_LITE_CFG``, ``NVFP4_AWQ_CLIP_CFG``) the
oracle's ``fake_quant_nvfp4`` stands in for ``tensor_quant.dynamic_block_quantize_op``, as in
``tools/gen_awq_golden.py``.  Every preset listed in ``CASES`` runs through the reference this way; none had to be
pinned against the oracle instead.  A case whose export the reference refuses stores the exception instead of tensors.

Arrays (``<case>`` is a preset name or a ``MIXED_*`` name from ``MIXED``):
  base/param/<name>            raw bytes of every parameter of the un-quantized model (bf16);
  <case>/in/param/<name>       a parameter after calibration, only where it differs from ``base`` (AWQ-lite and
                               SmoothQuant rescale weights);
  <case>/in/q/<quantizer>.<b>  every quantizer's ``_amax`` / ``_global_amax`` / ``_pre_quant_scale`` (float32 values);
  <case>/in/qdtype             JSON {"<quantizer>.<b>": torch dtype of that buffer};
  <case>/fmt                   JSON {linear name: the reference's ``get_quantization_format``} before export;
  <case>/out/<key>             raw bytes of each tensor of ``model.safetensors``, only where they differ from
                               ``base/param/<key>`` (unquantized tensors are stored once);
  <case>/meta                  JSON {key: [dtype, shape]} for every tensor of ``model.safetensors``;
  <case>/cfg                   ``hf_quant_config.json``;
  <case>/error                 JSON [exception type, message] when the export raised.

The zip entries carry a fixed timestamp, so that a rerun writes identical bytes.
"""

from __future__ import annotations

import copy
import json
import os
import sys
import tempfile
import warnings
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402

NAME = "ref_export_formats"
PRESETS = ("FP8_PER_CHANNEL_PER_TOKEN_CFG", "INT8_DEFAULT_CFG", "INT8_SMOOTHQUANT_CFG", "INT8_WEIGHT_ONLY_CFG",
           "FP8_2D_BLOCKWISE_WEIGHT_ONLY_CFG", "MXFP8_DEFAULT_CFG", "MXFP4_DEFAULT_CFG", "MXFP4_MLP_WEIGHT_ONLY_CFG",
           "W4A8_MXFP4_FP8_CFG", "W4A8_NVFP4_FP8_CFG", "NVFP4_AWQ_LITE_CFG", "NVFP4_AWQ_CLIP_CFG",
           "NVFP4_MLP_ONLY_CFG", "NVFP4_OMLP_ONLY_CFG")
# mixed precision, written as quant_cfg lists: {case: [(pattern prefix, preset whose weight / input entries it takes)]},
# later entries win, as in any quant_cfg list
MIXED = {
    "MIXED_FP8_ATTN_NVFP4_MLP": [("*self_attn*", "FP8_DEFAULT_CFG"), ("*mlp*", "NVFP4_DEFAULT_CFG")],
    "MIXED_NVFP4_FP8PC_O_DOWN": [("*", "NVFP4_DEFAULT_CFG"), ("*o_proj*", "FP8_PER_CHANNEL_PER_TOKEN_CFG"),
                                 ("*down_proj*", "FP8_PER_CHANNEL_PER_TOKEN_CFG")],
}
CASES = PRESETS + tuple(MIXED)


def mixed_config(case: str, preset) -> dict:
    """The quant config of a ``MIXED`` case; ``preset(name)`` returns a preset dict (the reference's ``mtq`` configs
    or the mirror's ``config.get_preset``), whose ``quant_cfg`` starts with disable-all, the weight and the input
    entry, followed by the default-disabled entries."""
    entries = []
    tail = None
    for prefix, name in MIXED[case]:
        qc = copy.deepcopy(preset(name)["quant_cfg"])
        for e in qc:
            if e.get("quantizer_name") in ("*weight_quantizer", "*input_quantizer"):
                entries.append({**e, "quantizer_name": prefix + e["quantizer_name"].lstrip("*")})
        tail = qc[3:]
    return {"quant_cfg": [{"quantizer_name": "*", "enable": False}, *entries, *tail], "algorithm": "max"}


def tiny_llama_config():
    from transformers import LlamaConfig

    return LlamaConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                       num_key_value_heads=2, vocab_size=128, max_position_embeddings=128, tie_word_embeddings=False,
                       architectures=["LlamaForCausalLM"])


def raw(t):
    import torch

    t = t.detach().contiguous().reshape(-1)
    return t.view(torch.uint8).numpy().copy() if t.numel() else np.zeros(0, np.uint8)


def _fix_zip_times(path):
    """Rewrite an .npz with a fixed timestamp on every entry (np.savez stamps the current time)."""
    with zipfile.ZipFile(path) as z:
        items = [(i.filename, z.read(i)) for i in z.infolist()]
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name, data in items:
            info = zipfile.ZipInfo(name, date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, data)


def main(ref_root="/root/reference"):
    from oracle.gen_golden import _install_shim

    _install_shim()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    import torch
    from safetensors.torch import load_file
    from transformers import LlamaForCausalLM

    import modelopt.torch.quantization as mtq
    from modelopt.torch.export import export_hf_checkpoint
    from modelopt.torch.export.quant_utils import get_quantization_format
    from modelopt.torch.quantization import tensor_quant as ref_tensor_quant

    from tools.gen_awq_golden import _stand_in

    ref_tensor_quant.dynamic_block_quantize_op = _stand_in
    torch.set_num_threads(1)
    cfg = tiny_llama_config()
    cfg.dtype = torch.bfloat16
    torch.manual_seed(0)
    base = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    g = torch.Generator().manual_seed(1)
    data = [torch.randint(0, 128, (2, 48), generator=g) for _ in range(4)]

    out = {}
    base_raw = {name: raw(p) for name, p in base.named_parameters()}
    for name, r in base_raw.items():
        out[f"base/param/{name}"] = r
    for case in CASES:
        m = copy.deepcopy(base)
        qcfg = mixed_config(case, lambda n: getattr(mtq, n)) if case in MIXED else copy.deepcopy(getattr(mtq, case))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mtq.quantize(m, qcfg, lambda mm: [mm(d) for d in data])
        for name, p in m.named_parameters():
            r = raw(p)
            if not np.array_equal(r, base_raw[name]):
                out[f"{case}/in/param/{name}"] = r
        fmts, qdtype = {}, {}
        for name, mod in m.named_modules():
            if type(mod).__name__ in ("TensorQuantizer", "StaticBlockScaleQuantizer", "NVFP4StaticQuantizer"):
                for b in ("_amax", "_global_amax", "_pre_quant_scale"):
                    t = getattr(mod, b, None)
                    if isinstance(t, torch.Tensor):
                        out[f"{case}/in/q/{name}.{b}"] = t.detach().float().numpy().copy()
                        qdtype[f"{name}.{b}"] = str(t.dtype)
            if isinstance(mod, torch.nn.Linear) and hasattr(mod, "weight_quantizer"):
                fmts[name] = get_quantization_format(mod)
        out[f"{case}/in/qdtype"] = np.array(json.dumps(qdtype, sort_keys=True))
        out[f"{case}/fmt"] = np.array(json.dumps(fmts, sort_keys=True))
        with tempfile.TemporaryDirectory() as d:
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    export_hf_checkpoint(m, export_dir=d)
            except Exception as e:  # noqa: BLE001 -- recorded: the mirror must refuse the same way
                out[f"{case}/error"] = np.array(json.dumps([type(e).__name__, str(e)]))
                print("export", case, "raised", type(e).__name__, e)
                continue
            sd = load_file(os.path.join(d, "model.safetensors"))
            meta = {}
            for k, v in sorted(sd.items()):
                r = raw(v)
                if k not in base_raw or not np.array_equal(r, base_raw[k]):
                    out[f"{case}/out/{k}"] = r
                meta[k] = [str(v.dtype), list(v.shape)]
            out[f"{case}/meta"] = np.array(json.dumps(meta, sort_keys=True))
            with open(os.path.join(d, "hf_quant_config.json")) as f:
                out[f"{case}/cfg"] = np.array(json.dumps(json.load(f)))
        print("export", case, len(sd), "tensors", json.loads(str(out[f"{case}/cfg"]))["quantization"])
    golden.save(NAME, out)
    for p in sorted(os.listdir(golden.DIR)):
        if p.startswith(NAME + ".") and p.endswith(".npz"):
            _fix_zip_times(os.path.join(golden.DIR, p))
    print("wrote", NAME, len(out), "arrays")


if __name__ == "__main__":
    main(*sys.argv[1:])
