"""Which operand formats can the post-LN audio / text stacks afford?  (VERDICT r1 item 4.)

The CUDA path runs HuBERT / BERT products as three bf16 MMAs on (hi, lo) operand pairs (MER_GEMM_BF16X3, ~2^-17 per
operand).  This script measures, with the oracle on the CPU, what cheaper schemes would cost in accuracy at FULL depth
(12 layers), on the default and on the x5 stress checkpoint, by rounding the operands of every product the way each
scheme's tensor-core instruction would (accumulation stays fp32, as on the device):

  tf32 / f16   both operands to 11 significant bits (1 MMA at the tf32 / f16 rate)
  w11          activations exact, weights to 11 bits   = the best any TWO-term split can do: hi*hi + lo*hi recovers one
               operand, the other keeps its 11-bit (fp16) or 8-bit (bf16) rounding                       (2 MMAs)
  mixed        11-bit operands everywhere except the GEMMs that feed the residual stream (attention out-proj, FC2,
               conv6, feature projection), which stay exact                                              (1 and 3 MMAs)
  bf16x3       both operands to 16 significant bits (hi + lo), the lo*lo term dropped                   (3 MMAs)
  f16-layers   11-bit operands in the 12 transformer layers (62 % of HuBERT's flops, all of BERT's), bf16x3 in the
               convolutional feature encoder and the feature projection                                  (1 | 3 MMAs)
  f16-conv     the converse: 11-bit operands in conv1-6 only                                             (1 | 3 MMAs)

Attention operands (q, k, v, p) are rounded to 11 bits in every scheme except fp32, as the tensor-core attention kernels do.
Metric: the test metric of tests/ (max |feature - fp32 feature| / max |fp32 feature| on the UTTERANCE readout).
Writes profiles/r2_precision_table.json.  CPU only; ~2 minutes."""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mertools_b200 import synthetic as S  # noqa: E402
from oracle import encoders as E  # noqa: E402
from oracle import pipeline as P  # noqa: E402


def rnd(x, bits):
    """Round-to-nearest to `bits` significant bits (fp32 in, fp32 out)."""
    if bits >= 24:
        return x
    drop = 24 - bits
    i = x.contiguous().view(torch.int32)
    i = (i + (1 << (drop - 1))) & ~((1 << drop) - 1)
    return i.view(torch.float32)


class Shim:
    """torch.nn.functional as the oracle sees it, with operand rounding on linear / conv1d and on attention."""

    def __init__(self, mode):
        self.mode = mode
        self.residual_feeding = False
        self.in_layers = False   # set by the patched _linear: the product belongs to a transformer layer

    def bits(self):
        m = self.mode
        if m == "fp32":
            return 24, 24
        if m in ("tf32", "f16"):
            return 11, 11
        if m == "w11":
            return 24, 11
        if m == "bf16x3":
            return 16, 16
        if m == "mixed":
            return (24, 24) if self.residual_feeding else (11, 11)
        if m == "f16-layers":
            return (11, 11) if self.in_layers else (16, 16)
        if m == "f16-conv":
            return (16, 16) if self.in_layers else (11, 11)
        raise ValueError(m)

    def linear(self, x, w, b=None):
        ab, wb = self.bits()
        return TF.linear(rnd(x, ab), rnd(w, wb), b)

    def conv1d(self, x, w, b=None, **kw):
        self.in_layers = False
        if kw.get("groups", 1) > 1:      # the positional conv runs as an fp16 GEMM in every scheme of the product
            return TF.conv1d(rnd(x, 11), rnd(w, 11), b, **kw) if self.mode != "fp32" else TF.conv1d(x, w, b, **kw)
        ab, wb = self.bits()
        return TF.conv1d(rnd(x, ab), rnd(w, wb), b, **kw)

    def __getattr__(self, k):
        return getattr(TF, k)


def patched(mode):
    shim = Shim(mode)
    orig_linear, orig_mha, orig_F = E._linear, E._mha, E.F
    feeding = ("out_proj", "output_dense", "output.dense", "feature_projection.projection", "attention.output.dense")

    def linear(x, sd, prefix, dtype):
        shim.residual_feeding = any(prefix.endswith(f) for f in feeding)
        shim.in_layers = ".layers." in prefix or ".layer." in prefix
        return shim.linear(x, E._t(sd, prefix + ".weight", dtype), E._t(sd, prefix + ".bias", dtype))

    def mha(q, k, v, heads, bias=None):
        if mode == "fp32":
            return orig_mha(q, k, v, heads, bias)
        import math
        B, T, D = q.shape
        hd = D // heads
        q, k, v = (rnd(t, 11).view(B, T, heads, hd).transpose(1, 2) for t in (q, k, v))
        s = q @ k.transpose(-1, -2) / math.sqrt(hd)
        p = torch.softmax(s if bias is None else s + bias, dim=-1)
        return (rnd(p, 11) @ v).transpose(1, 2).reshape(B, T, D)

    class Ctx:
        def __enter__(self):
            E._linear, E._mha, E.F = linear, mha, shim

        def __exit__(self, *a):
            E._linear, E._mha, E.F = orig_linear, orig_mha, orig_F
    return Ctx()


def rel(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / np.abs(b).max())


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    modes = ["tf32", "w11", "mixed", "f16-layers", "f16-conv", "bf16x3"]
    mma = {"tf32": "1 (tf32 / f16 rate)", "w11": "2", "mixed": "1, and 3 on the residual-feeding GEMMs", "bf16x3": "3",
           "f16-layers": "1 in the transformer layers, 3 in the conv stack", "f16-conv": "1 in conv1-6, 3 in the layers"}
    wav = (S.synth_waves(1, 80000, seed=31).astype(np.float64) / 32768.0)[0]
    ids = np.random.default_rng(3).integers(5, 2629, 32).tolist()
    ids[0], ids[-1] = 2, 3
    rows = []
    for scale in (1.0, 5.0):
        sd_a = S.hubert_state_dict(seed=1, layers=12, scale=scale)
        sd_t = S.bert_state_dict(2629, seed=2, layers=12, scale=scale)
        with torch.no_grad():
            ref_a = P.audio_clip_features(sd_a, wav, layers=12)
            ref_t = P.text_clip_features(sd_t, ids, 1, -1, layers=12)
            for m in modes:
                with patched(m):
                    a = P.audio_clip_features(sd_a, wav, layers=12)
                    t = P.text_clip_features(sd_t, ids, 1, -1, layers=12)
                row = dict(weights=f"x{scale:g}", scheme=m, mmas_per_product=mma[m], hubert_readout_max_rel=rel(a, ref_a),
                           bert_readout_max_rel=rel(t, ref_t))
                row["passes_1e-3_with_2x_margin"] = bool(max(row["hubert_readout_max_rel"], row["bert_readout_max_rel"]) < 5e-4)
                rows.append(row)
                print(json.dumps(row), flush=True)
    out = dict(what=__doc__.split("\n\n")[0], note="CPU emulation through the oracle (operand rounding only; fp32 accumulation); "
               "the device-measured bf16x3 figures are 3.9e-5 (HuBERT) / 7.4e-5 (BERT) at the bench configuration "
               "(tests/test_bench_config_gpu.py)", rows=rows)
    json.dump(out, open(os.path.join(ROOT, "profiles", "r2_precision_table.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
