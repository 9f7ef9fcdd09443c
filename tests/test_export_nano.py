"""CPU test of the Nano checkpoint export (nano_b200/export_nano.py; SURVEY section 8 row f1).  A seeded tiny GPT in the reference's
module naming (tests/golden/make_golden.py:nano_export_weights) is exported by OUR exporter; the files must be byte-identical to what
the reference's own export.py wrote for the same weights (F32, Q80 and a LoRA plug-in; SHA-256 digests in tests/golden/export_nano.npz),
and the F32 file's logits (oracle) must equal the reference PyTorch model's forward pass stored beside them."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from conftest import GOLDEN  # noqa: E402
from nano_b200 import export_nano, modelfile as mf  # noqa: E402
from oracle import bindings as ob  # noqa: E402

sys.path.insert(0, GOLDEN)
from make_golden import NANO_EXPORT_CONFIG, NANO_EXPORT_LORA, NANO_EXPORT_SEQ, nano_export_tokenizer, nano_export_weights, sha  # noqa: E402
sys.path.remove(GOLDEN)

S = NANO_EXPORT_SEQ
GOLD = np.load(os.path.join(GOLDEN, "export_nano.npz"))


class TinyGPT:
    """What export_nano reads from a checkpoint's model: .config, .state_dict() (tied classifier: one tensor under both names)
    and the RoPE tables the model carries."""

    def __init__(self, sd):
        self.config = SimpleNamespace(**NANO_EXPORT_CONFIG)
        self._sd = {k: torch.from_numpy(v) for k, v in sd.items() if k != "output.weight"}
        self._sd["output.weight"] = self._sd["tok_embeddings.weight"]
        self.freqs_cos, self.freqs_sin = torch.from_numpy(GOLD["freqs_cos"]), torch.from_numpy(GOLD["freqs_sin"])

    def state_dict(self):
        return self._sd


def test_export_is_byte_identical_to_the_reference_exporter_and_matches_the_model(tmp_path):
    sd, _lora = nano_export_weights()
    m = TinyGPT(sd)
    ours = str(tmp_path / "ours.bin")
    export_nano.export_nano(m, ours, mf.QUANT_F32, tokenizer_config=nano_export_tokenizer())
    assert sha(open(ours, "rb").read()) == str(GOLD["f32_sha256"]), "F32 export differs from the reference exporter's file"

    want = GOLD["logits"]                                                          # the reference PyTorch model, positions 0..S-1
    toks = mf.teacher_tokens(S, NANO_EXPORT_CONFIG["vocab_size"])
    o = ob.NanoOracle(ours, S)
    got = np.stack([o.forward(int(toks[p]), p) for p in range(S)])
    o.close()
    err, scale = float(np.abs(got - want).max()), float(np.abs(want).max())
    print(f"exported F32 file vs the PyTorch model: max|dlogit| {err:.3e} (logit scale {scale:.2f})")
    assert err < 2e-4 * max(1.0, scale)

    oursq = str(tmp_path / "ours_q80.bin")
    export_nano.export_nano(m, oursq, mf.QUANT_Q80, 64, tokenizer_config=nano_export_tokenizer())
    assert sha(open(oursq, "rb").read()) == str(GOLD["q80_sha256"]), "Q80 export differs from the reference exporter's file"


def test_lora_export_is_byte_identical_and_the_reference_engine_reproduces_the_lora_model(tmp_path):
    """export.py:117-226 / infer.c:436-500: the plug-in file is byte-identical to the reference exporter's for the same LoRA
    state dict, so the reference engine (and this engine, tests/test_gpu_lora.py) reads exactly the branches the model has."""
    _sd, lora = nano_export_weights()
    rank, alpha = NANO_EXPORT_LORA
    ours = str(tmp_path / "lora_ours.bin")
    info = export_nano.export_lora({k: torch.from_numpy(v) for k, v in lora.items()}, rank, alpha, SimpleNamespace(**NANO_EXPORT_CONFIG), ours)
    c = NANO_EXPORT_CONFIG
    kv = c["n_kv_head"] * c["n_embd"] // c["n_head"]
    assert info["bytes"] == 256 + 4 * c["n_layer"] * rank * (4 * c["n_embd"] + 2 * c["n_embd"] + 2 * kv)
    assert sha(open(ours, "rb").read()) == str(GOLD["lora_sha256"]), "LoRA export differs from the reference exporter's file"
