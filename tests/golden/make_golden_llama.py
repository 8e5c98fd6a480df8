"""Generate tests/golden/llama_text_golden.npz and the tokenizer fixture tests/golden/llama_tokenizer/ by running the
UNMODIFIED reference ``extract_embedding('llama-7b-hf', ..., gpu=-1)`` (MERBench/feature_extraction/text/
extract_text_huggingface.py) on CPU, for UTTERANCE and FRAME.

Run once in the build container (needs /root/reference, transformers and sentencepiece; NOT on the GPU box):
    python tests/golden/make_golden_llama.py
No LLaMA tokenizer is available offline, so a small one is trained: sentencepiece BPE on the Chinese column of the
reference's MER2023 transcription (vocab 4000, byte fallback, unk / bos / eos = 0 / 1 / 2, one thread), saved as
``tokenizer.model`` with a LlamaTokenizer ``tokenizer_config.json`` (BOS, no EOS: find_start_end_pos gives (1, None)).
The model is ``LlamaModel`` with mertools_b200.synthetic.llama_state_dict (hidden 512, 4 heads of 128, FFN 1408,
6 layers, max_position_embeddings 2048, rms_norm_eps 1e-6).  Stubs: a ``config`` module with patched paths.  No
reference source is copied.
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
TOK_DIR = os.path.join(OUT, "llama_tokenizer")
SEED = 21

from mertools_b200 import synthetic as S  # noqa: E402

TOKENIZER_CONFIG = {"tokenizer_class": "LlamaTokenizer", "add_bos_token": True, "add_eos_token": False,
                    "bos_token": "<s>", "eos_token": "</s>", "unk_token": "<unk>", "legacy": True,
                    "clean_up_tokenization_spaces": False, "model_max_length": 2048}


def llama_config(eps=1e-6):
    from transformers import LlamaConfig
    c = S.LLAMA_SMALL_CFG
    return LlamaConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], num_attention_heads=c["heads"],
                       intermediate_size=c["ffn"], num_hidden_layers=c["layers"],
                       max_position_embeddings=c["max_pos"], rms_norm_eps=eps)


def train_tokenizer(df, work):
    import sentencepiece as spm
    text = os.path.join(work, "chinese.txt")
    rows = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
    with open(text, "w", encoding="utf-8") as f:
        f.write("\n".join(rows) + "\n")
    spm.SentencePieceTrainer.train(input=text, model_prefix=os.path.join(work, "sp"), model_type="bpe",
                                   vocab_size=S.LLAMA_SMALL_CFG["vocab"], byte_fallback=True, unk_id=0, bos_id=1,
                                   eos_id=2, pad_id=-1, num_threads=1, character_coverage=1.0)
    os.makedirs(TOK_DIR, exist_ok=True)
    shutil.copy(os.path.join(work, "sp.model"), os.path.join(TOK_DIR, "tokenizer.model"))
    with open(os.path.join(TOK_DIR, "tokenizer_config.json"), "w") as f:
        json.dump(TOKENIZER_CONFIG, f, indent=1)
    print(f"tokenizer: {len(rows)} rows")


def main():
    import pandas as pd
    from transformers import AutoTokenizer, LlamaModel
    work = tempfile.mkdtemp(prefix="mer_golden_llama_")
    df = pd.read_csv(os.path.join(REF, "dataset", "mer2023-dataset-process", "transcription-engchi-polish.csv"))
    train_tokenizer(df, work)

    cfg = types.ModuleType("config")
    feats = os.path.join(work, "features")
    cfg.PATH_TO_TRANSCRIPTIONS = {"MER2023": os.path.join(work, "transcription.csv")}
    cfg.PATH_TO_FEATURES = {"MER2023": feats}
    cfg.PATH_TO_PRETRAINED_MODELS = os.path.join(work, "tools")
    sys.modules["config"] = cfg
    mdir = os.path.join(work, "tools", "transformers", "llama-7b-hf")
    m = LlamaModel(llama_config())
    m.load_state_dict({k: torch.from_numpy(v) for k, v in S.llama_state_dict(seed=SEED).items()}, strict=True)
    m.save_pretrained(mdir)
    for f in os.listdir(TOK_DIR):
        shutil.copy(os.path.join(TOK_DIR, f), mdir)
    tok = AutoTokenizer.from_pretrained(mdir, use_fast=False)

    # rows: ordinary sentences, the longest one of the corpus (> 64 tokens), an empty (NaN) row (the zeros rule), a
    # blank that tokenises to BOS + one piece and a one-character sentence (a single kept token: no mean at UTTERANCE)
    chin = [s for s in df["chinese"] if isinstance(s, str) and len(s) > 0]
    longest = max(chin, key=lambda s: len(tok(s)["input_ids"]))
    sents = chin[:5] + [longest, np.nan, " ", chin[5][:1], chin[6]]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    pd.DataFrame({"name": names, "chinese": sents, "english": ["x"] * len(sents)}).to_csv(
        cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], index=False)

    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ref_text", os.path.join(REF, "feature_extraction", "text", "extract_text_huggingface.py"))
    ref_text = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_text)
    out = {}
    for level in ("UTTERANCE", "FRAME"):
        ref_text.extract_embedding("llama-7b-hf", cfg.PATH_TO_TRANSCRIPTIONS["MER2023"], feats, level, gpu=-1)
        sd = os.path.join(feats, f"llama-7b-hf-{level[:3]}")
        for i, name in enumerate(names):
            out[f"{level[:3].lower()}{i}"] = np.load(os.path.join(sd, f"{name}.npy"))
    ids = {f"ids{i}": np.array(tok(s)["input_ids"], np.int64) for i, s in enumerate(sents) if isinstance(s, str)}
    start, end = ref_text.find_start_end_pos(tok)
    np.savez_compressed(os.path.join(OUT, "llama_text_golden.npz"), seed=SEED, start=start,
                        end=0 if end is None else end,  # 0: None (no end token) row_names=np.array(names),
                        sentences=np.array([s if isinstance(s, str) else "" for s in sents]),
                        isnan=np.array([not isinstance(s, str) for s in sents]), **ids, **out)
    print("llama text:", {k: (v.shape, v.dtype) for k, v in out.items()}, "lens", [len(v) for v in ids.values()])
    shutil.rmtree(work)


if __name__ == "__main__":
    main()
