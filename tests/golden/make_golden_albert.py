"""Generate tests/golden/albert_text_golden.npz and the tokenizer fixture tests/golden/albert_tokenizer/ by running the
UNMODIFIED reference ``extract_embedding`` (MERBench/feature_extraction/text/extract_text_huggingface.py) on CPU, for
UTTERANCE and FRAME, on three synthetic checkpoints:

- ``tiny``: ``albert_chinese_tiny`` (AutoModel + BertTokenizer, :164-166) on the Chinese column: 312 wide, 12 heads of
  26 (padded to 32 on the device), FFN 1248, 4 layers, gelu, BertTokenizer over tests/golden/text_vocab.txt;
- ``small``: ``albert_chinese_small``, the same branch: 384 wide, 12 heads of 32, FFN 1536, 4 layers, gelu;
- ``base``: ``albert-base-v2`` with language='english' (the ``-langeng-`` save dir) on the English column, through the
  AutoModel + AutoTokenizer(use_fast=False) branch: 768 wide, 12 heads, FFN 3072, 3 layers (hidden state 0, the mapped
  embedding, enters the readout), gelu_new.

No ALBERT vocabulary is available offline, so the English one is trained: a sentencepiece unigram model on both columns
of the reference's MER2023 transcription (vocab 4000, ALBERT's ids <pad> = 0, <unk> = 1, [CLS] = 2, [SEP] = 3, [MASK] = 4,
one thread), saved as ``spiece.model`` with an AlbertTokenizer ``tokenizer_config.json``.  Configs:
mertools_b200.synthetic.ALBERT_GOLDEN_CFGS; weights: synthetic.albert_state_dict (seed stored).  Keys are
``<family>_<name>`` as in xlnet_text_golden.npz: FRAME features keep every FRAME_STEP-th token row (``fra{i}``) and
``fran{i}`` records the reference's row count; ``utt{i}`` is whole; ``ids{i}`` holds the tokenizer's input_ids.

Run once in the build container (needs /root/reference, transformers and sentencepiece; NOT on the GPU box):
    python tests/golden/make_golden_albert.py
Stubs: a ``config`` module with patched paths.  No reference source is copied.
"""
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
TOK_DIR = os.path.join(OUT, "albert_tokenizer")
SEEDS = {"tiny": 43, "small": 45, "base": 47}
NAMES = {"tiny": ("albert_chinese_tiny", "chinese"), "small": ("albert_chinese_small", "chinese"),
         "base": ("albert-base-v2", "english")}
VOCAB = 4000
FRAME_STEP = 4
TOKENIZER_CONFIG = {"tokenizer_class": "AlbertTokenizer"}

from mertools_b200 import synthetic as S  # noqa: E402


def train_tokenizer(df, work):
    import sentencepiece as spm
    text = os.path.join(work, "text.txt")
    rows = [s for col in ("chinese", "english") for s in df[col] if isinstance(s, str) and len(s) > 0]
    with open(text, "w", encoding="utf-8") as f:
        f.write("\n".join(rows) + "\n")
    spm.SentencePieceTrainer.train(input=text, model_prefix=os.path.join(work, "sp"), model_type="unigram",
                                   vocab_size=VOCAB, pad_id=0, unk_id=1, bos_id=-1, eos_id=-1, num_threads=1,
                                   user_defined_symbols=["[CLS]", "[SEP]", "[MASK]"])
    os.makedirs(TOK_DIR, exist_ok=True)
    shutil.copy(os.path.join(work, "sp.model"), os.path.join(TOK_DIR, "spiece.model"))
    with open(os.path.join(TOK_DIR, "tokenizer_config.json"), "w") as f:
        json.dump(TOKENIZER_CONFIG, f, indent=1)
    print(f"tokenizer: {len(rows)} rows")


def main():
    import pandas as pd
    import transformers as tf
    work = tempfile.mkdtemp(prefix="mer_golden_albert_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))
    train_tokenizer(df, work)
    vocab_file = os.path.join(OUT, "text_vocab.txt")
    bert_vocab = len(open(vocab_file, encoding="utf-8").read().splitlines())

    cfg = types.ModuleType("config")
    cfg.PATH_TO_TRANSCRIPTIONS = {"MER2023": os.path.join(work, "transcription.csv")}
    sys.modules["config"] = cfg
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ref_text", os.path.join(REF, "feature_extraction", "text", "extract_text_huggingface.py"))
    ref_text = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_text)

    out = {}
    for family in ("tiny", "small", "base"):
        name, lang = NAMES[family]
        tools = os.path.join(work, family, "tools")
        feats = os.path.join(work, family, "features")
        cfg.PATH_TO_PRETRAINED_MODELS = tools
        mdir = os.path.join(tools, "transformers", name)
        vocab = VOCAB if family == "base" else bert_vocab
        kw = dict(S.ALBERT_GOLDEN_CFGS[family], vocab_size=vocab)
        m = tf.AlbertModel(tf.AlbertConfig(**kw))
        m.load_state_dict({k: torch.from_numpy(v) for k, v in S.albert_state_dict(kw, SEEDS[family]).items()},
                          strict=True)
        m.save_pretrained(mdir)
        if family == "base":
            shutil.copy(os.path.join(TOK_DIR, "spiece.model"), mdir)
            shutil.copy(os.path.join(TOK_DIR, "tokenizer_config.json"), mdir)
            tok = tf.AutoTokenizer.from_pretrained(mdir, use_fast=False)
        else:
            tf.BertTokenizer(vocab_file).save_pretrained(mdir)
            tok = tf.BertTokenizer.from_pretrained(mdir, use_fast=False)
        # rows: ordinary sentences, the longest one of the column (> 64 tokens: crosses two key tiles), an empty (NaN)
        # row (the zeros rule), a blank (specials only: the zeros rule too) and a one-character sentence
        col = [s for s in df[lang] if isinstance(s, str) and len(s) > 0]
        longest = max(col, key=lambda s: len(tok(s)["input_ids"]))
        assert len(tok(longest)["input_ids"]) > 64, len(tok(longest)["input_ids"])
        sents = col[:5] + [longest, np.nan, " ", col[5][:1], col[6]]
        names = [f"sample_{i:05d}" for i in range(len(sents))]
        pd.DataFrame({"name": names, "chinese": sents if lang == "chinese" else ["x"] * len(sents),
                      "english": sents if lang == "english" else ["x"] * len(sents)}).to_csv(
            cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)
        for level in ("UTTERANCE", "FRAME"):
            ref_text.extract_embedding(name, cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1,
                                       language=lang)
            sd = os.path.join(feats, f"{name}-{'langeng-' if lang == 'english' else ''}{level[:3]}")
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
                    f"{family}_end": end,
                    f"{family}_sentences": np.array([s if isinstance(s, str) else "" for s in sents]),
                    f"{family}_isnan": np.array([not isinstance(s, str) for s in sents])})
        print(family, "lens", [len(out[k]) for k in out if k.startswith(f"{family}_ids")])
    np.savez_compressed(os.path.join(OUT, "albert_text_golden.npz"), **out)
    shutil.rmtree(work)
    print("transformers", tf.__version__, "torch", torch.__version__)


if __name__ == "__main__":
    main()
