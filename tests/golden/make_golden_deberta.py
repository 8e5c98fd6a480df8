"""Generate tests/golden/deberta_text_golden.npz by running the UNMODIFIED reference
``extract_embedding('deberta-chinese-large', ..., gpu=-1)`` (MERBench/feature_extraction/text/
extract_text_huggingface.py) on CPU, for UTTERANCE and FRAME, on two synthetic checkpoints:

- ``v1``: a DebertaModel shaped as deberta-large (relative attention over max_relative_positions, c2p | p2c, no
  absolute positions, no token types) at width 768 / 12 heads, 4 layers;
- ``v2``: a DebertaV2Model shaped as deberta-v2-xlarge (log position buckets, LayerNorm'd relative table,
  share_att_key, the conv layer after layer 0) at width 512 / 8 heads, 5 layers, so that hs[1] (the conv output)
  enters the last-four readout.

Configs: mertools_b200.synthetic.DEBERTA_GOLDEN_CFGS; weights: synthetic.deberta_state_dict (seed stored).  The
reference loads this model name with BertTokenizer (:164-166); the vocabulary is the committed synthetic
tests/golden/text_vocab.txt of make_golden.py.  Keys are ``<family>_<name>`` with the names of the other text goldens,
except that FRAME features keep every FRAME_STEP-th token row (``fra{i}``, fixture size, as audio_golden.npz does) and
``fran{i}`` records the reference's row count; the UTTERANCE features (``utt{i}``, the mean over all rows) are whole.

Run once in the build container (needs /root/reference and transformers; NOT on the GPU box):
    python tests/golden/make_golden_deberta.py
Stubs: a ``config`` module with patched paths.  No reference source is copied.
"""
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference/MERBench"
OUT = os.path.dirname(os.path.abspath(__file__))
SEEDS = {"v1": 27, "v2": 29}
NAME = "deberta-chinese-large"
FRAME_STEP = 4

from mertools_b200 import synthetic as S  # noqa: E402


def main():
    import pandas as pd
    import transformers as tf
    work = tempfile.mkdtemp(prefix="mer_golden_deberta_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))
    vocab_file = os.path.join(OUT, "text_vocab.txt")
    vocab = len(open(vocab_file, encoding="utf-8").read().splitlines())

    cfg = types.ModuleType("config")
    cfg.PATH_TO_TRANSCRIPTIONS = {"MER2023": os.path.join(work, "transcription.csv")}
    sys.modules["config"] = cfg
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ref_text", os.path.join(REF, "feature_extraction", "text", "extract_text_huggingface.py"))
    ref_text = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_text)

    out = {}
    for family in ("v1", "v2"):
        v2 = family == "v2"
        tools = os.path.join(work, family, "tools")
        feats = os.path.join(work, family, "features")
        cfg.PATH_TO_PRETRAINED_MODELS = tools
        mdir = os.path.join(tools, "transformers", NAME)
        kw = dict(S.DEBERTA_GOLDEN_CFGS[family], vocab_size=vocab)
        m = (tf.DebertaV2Model if v2 else tf.DebertaModel)((tf.DebertaV2Config if v2 else tf.DebertaConfig)(**kw))
        m.load_state_dict({k: torch.from_numpy(v) for k, v in S.deberta_state_dict(kw, v2, SEEDS[family]).items()},
                          strict=True)
        m.save_pretrained(mdir)
        tok = tf.BertTokenizer(vocab_file)
        tok.save_pretrained(mdir)
        # rows: ordinary sentences, the longest one of the corpus (> 64 tokens: crosses a key tile), an empty (NaN) row
        # (the zeros rule), a blank and a one-character sentence
        chin = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
        longest = max(chin, key=len)
        sents = chin[:5] + [longest, np.nan, " ", chin[5][:1], chin[6]]
        names = [f"sample_{i:05d}" for i in range(len(sents))]
        pd.DataFrame({"name": names, "chinese": sents, "english": ["x"] * len(sents)}).to_csv(
            cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)
        for level in ("UTTERANCE", "FRAME"):
            ref_text.extract_embedding(NAME, cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1)
            sd = os.path.join(feats, f"{NAME}-{level[:3]}")
            for i, row in enumerate(names):
                x = np.load(os.path.join(sd, f"{row}.npy"))
                if level == "FRAME":
                    out[f"{family}_fran{i}"] = x.shape[0]
                    x = x[::FRAME_STEP]
                out[f"{family}_{level[:3].lower()}{i}"] = x
        for i, s in enumerate(sents):
            if isinstance(s, str):
                out[f"{family}_ids{i}"] = np.array(tok(s)["input_ids"], np.int64)
        start, end = ref_text.find_start_end_pos(tok)
        out.update({f"{family}_seed": SEEDS[family], f"{family}_vocab_size": vocab, f"{family}_start": start,
                    f"{family}_end": end, f"{family}_sentences": np.array([s if isinstance(s, str) else "" for s in sents]),
                    f"{family}_isnan": np.array([not isinstance(s, str) for s in sents])})
        print(family, "lens", [len(out[k]) for k in out if k.startswith(f"{family}_ids")])
    np.savez_compressed(os.path.join(OUT, "deberta_text_golden.npz"), **out)
    shutil.rmtree(work)
    print("transformers", tf.__version__, "torch", torch.__version__)


if __name__ == "__main__":
    main()
