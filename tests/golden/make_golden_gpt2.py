"""Generate tests/golden/gpt2_chinese_text_golden.npz and tests/golden/wenzhong_text_golden.npz by running the UNMODIFIED
reference ``extract_embedding('gpt2-chinese-cluecorpussmall' | 'wenzhong2-gpt2-chinese', ..., gpu=-1)``
(MERBench/feature_extraction/text/extract_text_huggingface.py) on CPU, for UTTERANCE and FRAME.

Run once in the build container (needs /root/reference and transformers; NOT on the GPU box):
    python tests/golden/make_golden_gpt2.py
Tokenizers, from fixtures already committed, with the tokenizer configs of tests/golden/gpt2_tokenizer_configs.json:
- gpt2-chinese-cluecorpussmall: BertTokenizer over tests/golden/text_vocab.txt ([PAD] = 0).  It returns
  token_type_ids (all zero), which the reference passes on to GPT2Model, so every token also gets wte[0] added; the
  synthetic wte row 0 is not zero, so the goldens pin that term.  find_start_end_pos gives (1, -1).
- wenzhong2-gpt2-chinese: GPT2Tokenizer over the byte-level BPE of tests/golden/opt_tokenizer (vocab.json + merges.txt),
  adding no BOS and returning no token types: (0, None).
Models: ``GPT2Model`` with mertools_b200.synthetic.gpt2_state_dict at synthetic.GPT2_GOLDEN_CFGS (head_dim 64: hidden
256, 4 heads, FFN 1024; head_dim 96: hidden 768, 8 heads, FFN 3072; 6 layers each), saved with save_pretrained and run in
fp32 as the reference runs them.  Stubs: a ``config`` module with patched paths.  No reference source is copied.
"""
import gzip
import json
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
GOLDEN = {"gpt2-chinese-cluecorpussmall": "gpt2_chinese_text_golden.npz",
          "wenzhong2-gpt2-chinese": "wenzhong_text_golden.npz"}

from mertools_b200 import synthetic as S  # noqa: E402


def config(name):
    from transformers import GPT2Config
    c = S.GPT2_GOLDEN_CFGS[name]
    ids = dict(bos_token_id=2, eos_token_id=3, pad_token_id=0) if name == "gpt2-chinese-cluecorpussmall" else \
        dict(bos_token_id=2, eos_token_id=2, pad_token_id=1)
    return GPT2Config(vocab_size=c["vocab"], n_positions=c["max_pos"], n_embd=c["hidden"], n_layer=c["layers"],
                      n_head=c["heads"], n_inner=c["ffn"], **ids)


def state_dict(name, scale=1.0):
    c = S.GPT2_GOLDEN_CFGS[name]
    return S.gpt2_state_dict(seed=c["seed"], vocab=c["vocab"], hidden=c["hidden"], ffn=c["ffn"], layers=c["layers"],
                             max_pos=c["max_pos"], scale=scale)


def install_tokenizer(name, dest):
    """The committed tokenizer fixture of ``name`` in a model directory ``dest``."""
    os.makedirs(dest, exist_ok=True)
    if name == "gpt2-chinese-cluecorpussmall":
        shutil.copyfile(os.path.join(OUT, "text_vocab.txt"), os.path.join(dest, "vocab.txt"))
    else:
        for f in ("vocab.json", "merges.txt"):
            with gzip.open(os.path.join(OUT, "opt_tokenizer", f + ".gz"), "rb") as a, \
                    open(os.path.join(dest, f), "wb") as b:
                b.write(a.read())
    with open(os.path.join(OUT, "gpt2_tokenizer_configs.json")) as f:
        cfg = json.load(f)[name]
    with open(os.path.join(dest, "tokenizer_config.json"), "w") as f:
        json.dump(cfg, f, indent=1)


def main():
    import pandas as pd
    from transformers import GPT2Model
    work = tempfile.mkdtemp(prefix="mer_golden_gpt2_")
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

    for name, fn in GOLDEN.items():
        mdir = os.path.join(work, "tools", "transformers", name)
        m = GPT2Model(config(name))
        m.load_state_dict({k: torch.from_numpy(v) for k, v in state_dict(name).items()}, strict=True)
        m.save_pretrained(mdir)
        install_tokenizer(name, mdir)
        from mertools_b200.extract.text import _gpt2_tokenizer
        tok = _gpt2_tokenizer(name, mdir)
        assert len(tok) == S.GPT2_GOLDEN_CFGS[name]["vocab"], len(tok)
        # rows: ordinary sentences, the longest one of the corpus (> 64 tokens: crosses a key tile), an empty (NaN) row
        # (the zeros rule), a blank and a one-character sentence
        chin = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
        longest = max(chin, key=lambda s: len(tok(s)["input_ids"]))
        sents = chin[:5] + [longest, np.nan, " ", chin[5][:1], chin[6]]
        names = [f"sample_{i:05d}" for i in range(len(sents))]
        pd.DataFrame({"name": names, "chinese": sents, "english": ["x"] * len(sents)}).to_csv(
            cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)
        out = {}
        for level in ("UTTERANCE", "FRAME"):
            ref_text.extract_embedding(name, cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1)
            sd = os.path.join(feats, f"{name}-{level[:3]}")
            for i, row in enumerate(names):
                out[f"{level[:3].lower()}{i}"] = np.load(os.path.join(sd, f"{row}.npy"))
        ids, tts = {}, {}
        for i, s in enumerate(sents):
            if isinstance(s, str):
                enc = tok(s)
                ids[f"ids{i}"] = np.array(enc["input_ids"], np.int64)
                if "token_type_ids" in enc:
                    tts[f"types{i}"] = np.array(enc["token_type_ids"], np.int64)
        start, end = ref_text.find_start_end_pos(tok)
        np.savez_compressed(os.path.join(OUT, fn), seed=S.GPT2_GOLDEN_CFGS[name]["seed"], start=start,
                            end=0 if end is None else end,  # 0: None (no end token)
                            sentences=np.array([s if isinstance(s, str) else "" for s in sents]),
                            isnan=np.array([not isinstance(s, str) for s in sents]), **ids, **tts, **out)
        print(f"{name}:", {k: (v.shape, v.dtype) for k, v in out.items()}, "lens", [len(v) for v in ids.values()],
              "token types:", bool(tts))
    shutil.rmtree(work)


if __name__ == "__main__":
    main()
