"""Which operand format should the EVA02 tower (eva02_base_patch14_224, MER_VISION_EVA02) default to?

An emulation of the device's operand formats through the float64 restatement (tests/_eva02_ref.py: operand rounding
only, accumulation exact), 12 blocks, 4 synthetic 112 x 112 faces through the host transform, on the default and the
x5 stress checkpoint:

  f16   both operands of every linear layer of the blocks to fp16
  tf32  both operands to tf32 (round-to-nearest, 10 mantissa bits)

In both, q | k (after the rotation), V and the attention probabilities are fp16: at 257 tokens attention takes the
fp16 V^T kernel whatever the stack's format.  Metric: max |feature - float64 feature| / max |float64 feature| over the
frame features (the golden tests' metric).  "f16" becomes Eva02Encoder's default if, on both checkpoints, its error is
within 10% of tf32's (the two formats carry the same 10-bit mantissa, and the fp16 attention operands are common to
both) and on the default checkpoint below the 1e-3 bar; fp16 then halves the operand bytes at twice the tensor rate.
Writes profiles/eva02_precision_table.json.  CPU only; a few minutes."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import _eva02_ref as R  # noqa: E402
import timm_eva_shim as T  # noqa: E402

from mertools_b200 import encoders as E  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    tf = T.create_transform(**T.resolve_model_data_config(T.Eva(depth=0)))
    px = R.pixels_from_frames(R.synth_faces(4, 112, 112, seed=9), tf)
    rows = []
    for weights, seed, scale in (("x1", 27, 1.0), ("x5", 28, 5.0)):
        lay = E.eva02_to_clip_layout(S.eva02_state_dict(seed, layers=12, scale=scale))
        ref = R.forward(lay, px)
        for scheme, op in (("f16", R.f16), ("tf32", R.tf32)):
            got = R.forward(lay, px, op=op)
            err = float((got - ref).abs().max() / ref.abs().max())
            rows.append(dict(model="eva02_base_patch14_224", weights=weights, scheme=scheme, layers=12,
                             readout_max_rel=err))
            print(rows[-1], flush=True)
    err = {(r["weights"], r["scheme"]): r["readout_max_rel"] for r in rows}
    f16_default = err["x1", "f16"] < 1e-3 and all(err[w, "f16"] <= 1.1 * err[w, "tf32"] for w in ("x1", "x5"))
    out = dict(what="Which operand format should the EVA02 tower default to?",
               note="CPU emulation through tests/_eva02_ref.py (operand rounding only; exact accumulation)",
               rows=rows, f16_default=f16_default)
    path = os.path.join(ROOT, "profiles", "eva02_precision_table.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(f"wrote {path}: f16_default={f16_default}")


if __name__ == "__main__":
    main()
