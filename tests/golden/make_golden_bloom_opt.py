"""Generate tests/golden/{bloom,opt}_text_golden.npz and the tokenizer fixtures tests/golden/{bloom,opt}_tokenizer/ by
running the UNMODIFIED reference ``extract_embedding('bloom-7b1' | 'opt-13b', ..., gpu=-1)`` (MERBench/
feature_extraction/text/extract_text_huggingface.py) on CPU, for UTTERANCE and FRAME.

Run once in the build container (needs /root/reference, transformers and tokenizers; NOT on the GPU box):
    python tests/golden/make_golden_bloom_opt.py
No BLOOM / OPT tokenizer is available offline, so one byte-level BPE is trained with ``tokenizers`` on the Chinese
column of the reference's MER2023 transcription (vocab 4000; specials <s> <pad> </s> <unk> = 0 1 2 3; one thread) and
saved twice: ``tokenizer.json`` for BLOOM (no BOS: find_start_end_pos gives (0, None)) and ``vocab.json`` +
``merges.txt`` with a GPT2Tokenizer config that adds a BOS (</s>, as OPT's does: (1, None)).  The vocabulary files are
committed gzip-compressed (``*.gz``, fixed mtime); ``unpack_tokenizer`` writes a loadable tokenizer directory.  The configs' bos / eos /
pad ids are the tokenizer's.  The models are ``BloomModel`` / ``OPTModel`` with mertools_b200.synthetic.
bloom_state_dict / opt_state_dict (hidden 512, 4 heads of 128, FFN 2048, 6 layers), saved with save_pretrained.
Stubs: a ``config`` module with patched paths.  No reference source is copied.
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
SEEDS = {"bloom": 23, "opt": 25}
NAMES = {"bloom": "bloom-7b1", "opt": "opt-13b"}
SPECIALS = ["<s>", "<pad>", "</s>", "<unk>"]

from mertools_b200 import synthetic as S  # noqa: E402

TOKENIZER_CONFIGS = {
    "bloom": {"tokenizer_class": "BloomTokenizer", "bos_token": "<s>", "eos_token": "</s>", "unk_token": "<unk>",
              "pad_token": "<pad>", "padding_side": "left", "model_max_length": 2048,
              "clean_up_tokenization_spaces": False},
    "opt": {"tokenizer_class": "GPT2Tokenizer", "add_bos_token": True, "bos_token": "</s>", "eos_token": "</s>",
            "unk_token": "</s>", "pad_token": "<pad>", "model_max_length": 2048, "errors": "replace",
            "clean_up_tokenization_spaces": False},
}


def config(family):
    from transformers import BloomConfig, OPTConfig
    c = S.LN_DECODER_SMALL_CFG
    if family == "bloom":
        return BloomConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], n_head=c["heads"], n_layer=c["layers"],
                           bos_token_id=0, eos_token_id=2, pad_token_id=1)
    return OPTConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], num_attention_heads=c["heads"], ffn_dim=c["ffn"],
                     num_hidden_layers=c["layers"], max_position_embeddings=c["max_pos"], word_embed_proj_dim=c["hidden"],
                     bos_token_id=2, eos_token_id=2, pad_token_id=1)


def state_dict(family, scale=1.0):
    c = S.LN_DECODER_SMALL_CFG
    if family == "bloom":
        return S.bloom_state_dict(seed=SEEDS["bloom"], vocab=c["vocab"], hidden=c["hidden"], layers=c["layers"],
                                  scale=scale)
    return S.opt_state_dict(seed=SEEDS["opt"], vocab=c["vocab"], hidden=c["hidden"], ffn=c["ffn"], layers=c["layers"],
                            max_pos=c["max_pos"], scale=scale)


def unpack_tokenizer(family, dest):
    """Write the committed tokenizer fixture of ``family`` as a loadable directory ``dest`` (``*.gz`` decompressed)."""
    src = os.path.join(OUT, f"{family}_tokenizer")
    os.makedirs(dest, exist_ok=True)
    for f in os.listdir(src):
        with (gzip.open if f.endswith(".gz") else open)(os.path.join(src, f), "rb") as a, \
                open(os.path.join(dest, f[:-3] if f.endswith(".gz") else f), "wb") as b:
            b.write(a.read())


def _gzip(path):
    with open(path, "rb") as a, open(path + ".gz", "wb") as raw, \
            gzip.GzipFile(filename="", mode="wb", fileobj=raw, mtime=0) as b:
        b.write(a.read())
    os.remove(path)


def train_tokenizer(df, work):
    os.environ["RAYON_NUM_THREADS"] = "1"
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, trainers
    rows = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    tok.train_from_iterator(rows, trainers.BpeTrainer(vocab_size=S.LN_DECODER_SMALL_CFG["vocab"], special_tokens=SPECIALS,
                                                      initial_alphabet=pre_tokenizers.ByteLevel.alphabet(),
                                                      show_progress=False))
    for family in ("bloom", "opt"):
        d = os.path.join(OUT, f"{family}_tokenizer")
        os.makedirs(d, exist_ok=True)
        if family == "bloom":
            tok.save(os.path.join(d, "tokenizer.json"))
            _gzip(os.path.join(d, "tokenizer.json"))
        else:
            tok.model.save(d)
            _gzip(os.path.join(d, "vocab.json"))
            _gzip(os.path.join(d, "merges.txt"))
        with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
            json.dump(TOKENIZER_CONFIGS[family], f, indent=1)
    print(f"tokenizer: {len(rows)} rows")


def main():
    import pandas as pd
    from transformers import AutoTokenizer, BloomModel, OPTModel
    work = tempfile.mkdtemp(prefix="mer_golden_bloom_opt_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))
    train_tokenizer(df, work)

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

    for family, cls in (("bloom", BloomModel), ("opt", OPTModel)):
        name = NAMES[family]
        mdir = os.path.join(work, "tools", "transformers", name)
        m = cls(config(family))
        m.load_state_dict({k: torch.from_numpy(v) for k, v in state_dict(family).items()}, strict=True)
        m.save_pretrained(mdir)
        unpack_tokenizer(family, mdir)
        tok = AutoTokenizer.from_pretrained(mdir, use_fast=False)
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
        ids = {f"ids{i}": np.array(tok(s)["input_ids"], np.int64) for i, s in enumerate(sents) if isinstance(s, str)}
        start, end = ref_text.find_start_end_pos(tok)
        np.savez_compressed(os.path.join(OUT, f"{family}_text_golden.npz"), seed=SEEDS[family], start=start,
                            end=0 if end is None else end,  # 0: None (no end token)
                            sentences=np.array([s if isinstance(s, str) else "" for s in sents]),
                            isnan=np.array([not isinstance(s, str) for s in sents]), **ids, **out)
        print(f"{family} text:", {k: (v.shape, v.dtype) for k, v in out.items()}, "lens",
              [len(v) for v in ids.values()])
    shutil.rmtree(work)


if __name__ == "__main__":
    main()
