"""Which operand format should the hidden-256 text stacks (ELECTRA-small, LERT-small) default to?

The emulation of scripts/precision_table.py (operand rounding of every product as the tensor-core instruction would do
it, fp32 accumulation, attention operands to 11 bits) at the two small shapes, 12 layers, on the default and the x5
stress checkpoint:

  f16      both operands of every product to 11 significant bits (one fp16 MMA per product)
  bf16x3   both operands to 16 significant bits (hi + lo), the lo*lo term dropped (three bf16 MMAs)

ELECTRA-small's embedding projection runs in the stack's format.  Metric: max |feature - fp32 feature| / max |fp32
feature| on the UTTERANCE readout (the tests' metric).  "f16" becomes BertEncoder's default at hidden 256 only if both
of its errors stay below 5e-4 (a 2x margin under the 1e-3 bar).  Writes profiles/electra_small_precision_table.json.
CPU only; about a minute."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _electra_ref import electra_features  # noqa: E402
from precision_table import patched, rel  # noqa: E402

from mertools_b200 import synthetic as S  # noqa: E402

SHAPES = ("chinese-electra-180g-small", "chinese-lert-small")


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    ids = np.random.default_rng(3).integers(5, 2629, 32).tolist()
    ids[0], ids[-1] = 2, 3
    rows = []
    for name in SHAPES:
        kw = dict(S.ELECTRA_PUBLISHED_CFGS[name], vocab_size=2629)
        for scale in (1.0, 5.0):
            sd = S.electra_state_dict(kw, seed=51, scale=scale)
            run = lambda: electra_features(sd, ids, kw["num_hidden_layers"], kw["num_attention_heads"])  # noqa: E731
            with torch.no_grad():
                ref = run()
                for m in ("f16", "bf16x3"):
                    with patched(m):
                        got = run()
                    row = dict(model=name, weights=f"x{scale:g}", scheme=m, layers=kw["num_hidden_layers"],
                               readout_max_rel=rel(got, ref))
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    f16_ok = all(r["readout_max_rel"] < 5e-4 for r in rows if r["scheme"] == "f16")
    out = dict(what=__doc__.split("\n\n")[0], note="CPU emulation through the oracle's helpers (operand rounding only; "
               "fp32 accumulation)", rows=rows, f16_default=f16_ok)
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "profiles", "electra_small_precision_table.json"), "w"), indent=1)
    print("default at hidden 256:", "f16" if f16_ok else "bf16x3")


if __name__ == "__main__":
    main()
