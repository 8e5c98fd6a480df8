"""Do fp16 operands hold the 1e-3 bar on whole audio clips, where the softmax runs over 1,250 .. 3,000 keys?

MER2023's extractor (extract/audio_mer2023.py) feeds each clip whole, with the readout hidden_states[-1].  The
emulation of scripts/precision_table.py (operand rounding of every product as the tensor-core instruction does it,
fp32 accumulation; q, k, v and the probabilities P rounded to 11 bits, as the fp16 V^T attention kernel does) on
HuBERT-base, 12 layers, the default and the x5 stress checkpoint, at clips of 1 s, 10 s, 25 s and 60 s:

  f16-layers  11-bit operands in the transformer layers (the default operand format of the post-LN family)
  bf16x3      16-bit operands everywhere

Metric: max |feature - fp32 feature| / max |fp32 feature|, on the UTTERANCE readout (the tests' metric) and on the
FRAME readout.  The question is whether the error GROWS with the row length: a default that depends on the row
length only helps if long rows are worse than the 10 s rows the fp16 path already serves.
Writes profiles/mer2023_long_audio_precision_table.json.  CPU only; a few minutes."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from precision_table import patched, rel  # noqa: E402

from mertools_b200 import synthetic as S  # noqa: E402
from oracle import encoders as E  # noqa: E402
from oracle import pipeline as P  # noqa: E402

SECONDS = (1, 10, 25, 60)


def last_hidden(sd, wav):
    iv = torch.from_numpy(P.wav2vec2_normalize(wav))[None]
    return E.hubert_hidden_states(sd, iv, layers=12)[-1][0].numpy()


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    rows = []
    for scale in (1.0, 5.0):
        sd = S.hubert_state_dict(seed=1, layers=12, scale=scale)
        for sec in SECONDS:
            wav = S.synth_waves(1, sec * 16000, seed=31 + sec)[0].astype(np.float64) / 32768.0
            with torch.no_grad():
                ref = last_hidden(sd, wav)
                for m in ("f16-layers", "bf16x3"):
                    with patched(m):
                        got = last_hidden(sd, wav)
                    row = dict(weights=f"x{scale:g}", seconds=sec, frames=int(ref.shape[0]), scheme=m,
                               utt_max_rel=rel(got.mean(axis=0), ref.mean(axis=0)), frame_max_rel=rel(got, ref))
                    rows.append(row)
                    print(json.dumps(row), flush=True)

    def worst(scheme, scale, long_rows):
        return max(r["utt_max_rel"] for r in rows if r["scheme"] == scheme and r["weights"] == scale
                   and (r["frames"] > 505) == long_rows)
    growth = {f"{m}_{w}": worst(m, w, True) / worst(m, w, False) for m in ("f16-layers", "bf16x3") for w in ("x1", "x5")}
    out = dict(what=__doc__.split("\n\n")[0], note="CPU emulation through the oracle (operand rounding only; fp32 "
               "accumulation); not a device measurement", rows=rows,
               long_over_short_worst_utt_error=growth)
    json.dump(out, open(os.path.join(ROOT, "profiles", "mer2023_long_audio_precision_table.json"), "w"), indent=1)
    print("worst UTT error, rows > 505 frames over rows <= 505 frames:", growth)


if __name__ == "__main__":
    main()
