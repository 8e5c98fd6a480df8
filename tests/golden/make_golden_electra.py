"""Generate tests/golden/electra_text_golden.npz by running the UNMODIFIED reference functions on CPU, on seeded synthetic
checkpoints (weights: mertools_b200.synthetic.electra_state_dict, configs: synthetic.ELECTRA_GOLDEN_CFGS, seeds stored):

- MERBench/feature_extraction/text/extract_text_huggingface.py ``extract_embedding``, UTTERANCE and FRAME, through its
  AutoModel + AutoTokenizer(use_fast=False) branch:
  - ``small``: ``chinese-electra-180g-small`` on the Chinese column: ElectraModel with the factorised 128-wide
    embedding projected to hidden 256, 4 heads of 64, FFN 1024, 5 layers;
  - ``base``: ``chinese-electra-180g-base``: embedding_size == hidden_size == 768, 4 layers;
  - ``lert_small``: ``chinese-lert-small``: a hidden-256 BertModel (4 heads, FFN 1024, 4 layers);
  - ``eng``: ``electra-base-discriminator`` with language='english' (the ``-langeng-`` save dir) on the English column,
    saved as ElectraForPreTraining so that the checkpoint carries the ``electra.`` prefix and the discriminator head.
  The tokenizer is BertTokenizer over tests/golden/text_vocab.txt.
- MER2023/feature_extraction/text/extract_text_embedding_LZ.py ``extract_bert_embedding_english`` (``words``):
  ``electra-base-discriminator`` (ElectraForPreTraining, base shape, 4 layers) over tests/golden/text_words_vocab.txt and
  the sentences of make_golden_words.py, FRAME and UTTERANCE.

Keys are ``<family>_<name>`` as in albert_text_golden.npz: FRAME features keep every FRAME_STEP-th token row (``fra{i}``)
and ``fran{i}`` records the reference's row count; ``utt{i}`` is whole; ``ids{i}`` holds the tokenizer's input_ids.

Run once in the build container (needs the reference sources and transformers; NOT on the GPU box):
    python tests/golden/make_golden_electra.py
Stubs: a ``config`` module with patched paths; for the word-level function, ``Module.to`` / ``BatchEncoding.to`` as
identities (it hard-codes cuda:N).  No reference source is copied.
"""
import importlib.util
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
REF_LZ = "/root/reference/MER2023/feature_extraction/text"
OUT = os.path.dirname(os.path.abspath(__file__))
SEEDS = {"small": 53, "base": 55, "lert_small": 57, "eng": 59, "words": 61}
NAMES = {"small": ("chinese-electra-180g-small", "chinese"), "base": ("chinese-electra-180g-base", "chinese"),
         "lert_small": ("chinese-lert-small", "chinese"), "eng": ("electra-base-discriminator", "english")}
CFG_OF = {"small": "small", "base": "base", "lert_small": "lert_small", "eng": "base", "words": "base"}
FRAME_STEP = 4
WORD_SENTENCES = {
    "clip0": "I'm really happy today, the movie was unbelievable! Did you like it?",
    "clip1": "No.",
    "clip2": "well it was okay I guess but the ending felt rushed and nobody laughed",
    "clip3": "Wow!!! Absolutely   fantastic, 10 out of 10.",
}

from mertools_b200 import synthetic as S  # noqa: E402


def _save_model(family, mdir, vocab):
    import transformers as tf
    kw = dict(S.ELECTRA_GOLDEN_CFGS[CFG_OF[family]], vocab_size=vocab)
    if family == "lert_small":
        kw = {k: v for k, v in kw.items() if k != "embedding_size"}
        m = tf.BertModel(tf.BertConfig(**kw), add_pooling_layer=False)
        sd = {k: v for k, v in S.electra_state_dict(dict(kw, embedding_size=kw["hidden_size"]), SEEDS[family]).items()}
    elif family in ("eng", "words"):
        m = tf.ElectraForPreTraining(tf.ElectraConfig(**kw))
        sd = S.electra_state_dict(kw, SEEDS[family], pretraining=True)
    else:
        m = tf.ElectraModel(tf.ElectraConfig(**kw))
        sd = S.electra_state_dict(kw, SEEDS[family])
    missing, unexpected = m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith(("position_ids", "token_type_ids")) for k in missing), (missing, unexpected)
    m.save_pretrained(mdir)


def _sentence_golden(out, ref_text, cfg, df, work, family):
    import pandas as pd
    import transformers as tf
    name, lang = NAMES[family]
    tools = os.path.join(work, family, "tools")
    feats = os.path.join(work, family, "features")
    cfg.PATH_TO_PRETRAINED_MODELS = tools
    mdir = os.path.join(tools, "transformers", name)
    vocab_file = os.path.join(OUT, "text_vocab.txt")
    vocab = len(open(vocab_file, encoding="utf-8").read().splitlines())
    _save_model(family, mdir, vocab)
    tf.BertTokenizer(vocab_file, do_lower_case=True).save_pretrained(mdir)
    tok = tf.AutoTokenizer.from_pretrained(mdir, use_fast=False)
    # rows: ordinary sentences, the longest one of the column (> 64 tokens: crosses two key tiles), an empty (NaN) row
    # (the zeros rule), a blank (specials only: the zeros rule too) and a one-character sentence
    col = [s for s in df[lang] if isinstance(s, str) and len(s) > 0]
    longest = max(col, key=lambda s: len(tok(s)["input_ids"]))
    assert len(tok(longest)["input_ids"]) > 64, len(tok(longest)["input_ids"])
    sents = col[:5] + [longest, np.nan, " ", col[5][:1], col[6]]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    pd.DataFrame({"name": names, "chinese": sents if lang == "chinese" else ["x"] * len(sents),
                  "english": sents if lang == "english" else ["x"] * len(sents)}).to_csv(
        cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)
    for level in ("UTTERANCE", "FRAME"):
        ref_text.extract_embedding(name, cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1, language=lang)
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
                f"{family}_end": end if end is not None else 0,
                f"{family}_sentences": np.array([s if isinstance(s, str) else "" for s in sents]),
                f"{family}_isnan": np.array([not isinstance(s, str) for s in sents])})
    print(family, "lens", [len(out[k]) for k in out if k.startswith(f"{family}_ids")])


def _word_golden(out, cfg, work):
    import pandas as pd
    import transformers as tf
    from transformers import BatchEncoding
    name = NAMES["eng"][0]
    mdir = os.path.join(work, "words", "tools", "transformers", name)
    vocab_file = os.path.join(OUT, "text_words_vocab.txt")
    vocab = len(open(vocab_file, encoding="utf-8").read().splitlines())
    _save_model("words", mdir, vocab)
    tf.BertTokenizer(vocab_file, do_lower_case=True).save_pretrained(mdir)
    cfg.PATH_TO_PRETRAINED_MODELS = os.path.join(work, "words", "tools")
    csv = os.path.join(work, "words", "trans.csv")
    pd.DataFrame({"name": list(WORD_SENTENCES), "sentence": list(WORD_SENTENCES.values())}).to_csv(csv, index=False)
    sys.path.insert(0, REF_LZ)
    spec = importlib.util.spec_from_file_location("ref_text_lz", os.path.join(REF_LZ, "extract_text_embedding_LZ.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    orig_mto, orig_bto = torch.nn.Module.to, BatchEncoding.to
    torch.nn.Module.to = lambda self, *a, **k: self
    BatchEncoding.to = lambda self, *a, **k: self
    try:
        for level in ("FRAME", "UTTERANCE"):
            sdir = os.path.join(work, "words", "feat")
            ref.extract_bert_embedding_english(name, csv, sdir, level, gpu=0)
            d = os.path.join(sdir, f"{name}-4-{level[:3]}")
            for clip in WORD_SENTENCES:
                out[f"words_{level[:3].lower()}_{clip}"] = np.load(os.path.join(d, f"{clip}.npy"))
    finally:
        torch.nn.Module.to, BatchEncoding.to = orig_mto, orig_bto
    out.update({"words_seed": SEEDS["words"], "words_vocab_size": vocab, "words_names": np.array(list(WORD_SENTENCES)),
                "words_sentences": np.array(list(WORD_SENTENCES.values()))})


def main():
    import pandas as pd
    import transformers as tf
    torch.manual_seed(0)
    work = tempfile.mkdtemp(prefix="mer_golden_electra_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))
    cfg = types.ModuleType("config")
    cfg.PATH_TO_TRANSCRIPTIONS = {"MER2023": os.path.join(work, "transcription.csv")}
    sys.modules["config"] = cfg
    spec = importlib.util.spec_from_file_location(
        "ref_text", os.path.join(REF, "feature_extraction", "text", "extract_text_huggingface.py"))
    ref_text = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_text)
    out = {}
    for family in ("small", "base", "lert_small", "eng"):
        _sentence_golden(out, ref_text, cfg, df, work, family)
    _word_golden(out, cfg, work)
    np.savez_compressed(os.path.join(OUT, "electra_text_golden.npz"), **out)
    shutil.rmtree(work)
    print("transformers", tf.__version__, "torch", torch.__version__)


if __name__ == "__main__":
    main()
