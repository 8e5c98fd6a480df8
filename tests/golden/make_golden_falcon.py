"""Generate tests/golden/falcon_text_golden.npz by running the UNMODIFIED reference
``extract_embedding('falcon-7b', ..., gpu=-1)`` (MERBench/feature_extraction/text/extract_text_huggingface.py) on CPU,
for UTTERANCE and FRAME.

Run once in the build container (needs /root/reference and transformers; NOT on the GPU box):
    python tests/golden/make_golden_falcon.py
The model is ``FalconModel`` (parallel attention, multi-query, no biases, rotary) with
mertools_b200.synthetic.falcon_state_dict at FALCON_SMALL_CFG (hidden 448 = 7 heads of 64, FFN 1792, 6 layers): hidden
and QKV width (576) are not multiples of 128, as falcon-7b's 4544 and 4672 are not, so the CUDA backend's padded
layout is exercised.  No Falcon tokenizer is available offline: the byte-level BPE of tests/golden/bloom_tokenizer
(tokenizer.json) is reused with tests/golden/falcon_tokenizer/tokenizer_config.json, which names
PreTrainedTokenizerFast as the published falcon-7b does and adds no BOS (find_start_end_pos gives (0, None)).  The
sentences are the BLOOM golden's rows.  Stubs: a ``config`` module with patched paths.  No reference source is copied.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/MERBench"
OUT = os.path.dirname(os.path.abspath(__file__))
SEED = 43
NAME = "falcon-7b"

from make_golden_bloom_opt import unpack_tokenizer  # noqa: E402

from mertools_b200 import synthetic as S  # noqa: E402


def config():
    from transformers import FalconConfig
    c = S.FALCON_SMALL_CFG
    return FalconConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], num_attention_heads=c["heads"],
                        ffn_hidden_size=c["ffn"], num_hidden_layers=c["layers"], max_position_embeddings=c["max_pos"],
                        layer_norm_epsilon=1e-5, bos_token_id=0, eos_token_id=2, pad_token_id=1)


def state_dict(scale=1.0):
    c = S.FALCON_SMALL_CFG
    return S.falcon_state_dict(seed=SEED, vocab=c["vocab"], hidden=c["hidden"], heads=c["heads"], ffn=c["ffn"],
                               layers=c["layers"], scale=scale)


def unpack_falcon_tokenizer(dest):
    """The BLOOM fixture's tokenizer.json with the Falcon tokenizer_config.json, as a loadable directory ``dest``."""
    unpack_tokenizer("bloom", dest)
    shutil.copy(os.path.join(OUT, "falcon_tokenizer", "tokenizer_config.json"), dest)


def main():
    import pandas as pd
    from transformers import AutoTokenizer, FalconModel
    work = tempfile.mkdtemp(prefix="mer_golden_falcon_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))

    cfg = types.ModuleType("config")
    feats = os.path.join(work, "features")
    cfg.PATH_TO_TRANSCRIPTIONS = {"MER2023": os.path.join(work, "transcription.csv")}
    cfg.PATH_TO_FEATURES = {"MER2023": feats}
    cfg.PATH_TO_PRETRAINED_MODELS = os.path.join(work, "tools")
    sys.modules["config"] = cfg
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ref_text", os.path.join(REF, "feature_extraction", "text", "extract_text_huggingface.py"))
    ref_text = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_text)

    mdir = os.path.join(work, "tools", "transformers", NAME)
    m = FalconModel(config())
    m.load_state_dict({k: torch.from_numpy(v) for k, v in state_dict().items()}, strict=True)
    m.save_pretrained(mdir)
    unpack_falcon_tokenizer(mdir)
    tok = AutoTokenizer.from_pretrained(mdir, use_fast=False)
    # the BLOOM golden's rows: ordinary sentences, the longest one of the corpus (> 64 tokens: crosses a key tile), an
    # empty (NaN) row (the zeros rule), a blank and a one-character sentence
    chin = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
    longest = max(chin, key=lambda s: len(tok(s)["input_ids"]))
    sents = chin[:5] + [longest, np.nan, " ", chin[5][:1], chin[6]]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    pd.DataFrame({"name": names, "chinese": sents, "english": ["x"] * len(sents)}).to_csv(
        cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)
    out = {}
    for level in ("UTTERANCE", "FRAME"):
        ref_text.extract_embedding(NAME, cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1)
        sd = os.path.join(feats, f"{NAME}-{level[:3]}")
        for i, row in enumerate(names):
            out[f"{level[:3].lower()}{i}"] = np.load(os.path.join(sd, f"{row}.npy"))
    ids = {f"ids{i}": np.array(tok(s)["input_ids"], np.int64) for i, s in enumerate(sents) if isinstance(s, str)}
    start, end = ref_text.find_start_end_pos(tok)
    np.savez_compressed(os.path.join(OUT, "falcon_text_golden.npz"), seed=SEED, start=start,
                        end=0 if end is None else end,  # 0: None (no end token)
                        sentences=np.array([s if isinstance(s, str) else "" for s in sents]),
                        isnan=np.array([not isinstance(s, str) for s in sents]), **ids, **out)
    print("falcon text:", {k: (v.shape, v.dtype) for k, v in out.items()}, "lens", [len(v) for v in ids.values()],
          "start/end", start, end)
    shutil.rmtree(work)


if __name__ == "__main__":
    main()
