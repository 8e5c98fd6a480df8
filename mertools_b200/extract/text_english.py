"""English word-aligned lexical features — H100 mirror of
MER2023/feature_extraction/text/extract_text_embedding_LZ.py:extract_bert_embedding_english (:168-311).

The host side is the reference's: split the transcript into words and sentences (:205-224), tokenise each
sentence as pre-split words (:232), and, after the encoder, merge sub-word embeddings back into one vector per
word (:254-291, ``combine_type`` mean | sum | last), then the FRAME / UTTERANCE save rules (:296-309).  The
encoder pass (sum of the last four hidden states of every real token, :236-238) runs in libmer_b200.so over
all sentences of a transcript as one packed batch.  BERT / RoBERTa / ELECTRA checkpoints only (the reference's list
also names ALBERT, XLNet, GPT, T5, DeBERTa, which this path does not run).
"""
from __future__ import annotations

import itertools
import os
import re
import time

import numpy as np


def split_words_and_sentences(sentence, lower):
    """Transcript -> list of sentences, each a list of cleaned words (:205-224)."""
    words = re.split(r"([ ,.!?])", sentence.strip())
    words = [w.strip().lower() for w in words if len(w.strip()) > 0]
    sentences, cur = [], []
    for word in words:
        if word in [".", "!", "?"]:
            if cur != []:
                sentences.append(cur)
                cur = []
        else:
            cleaned = re.sub(r"[^a-zA-Z0-9,.\'!?]+", "", word)
            if lower:
                cleaned = cleaned.lower()
            if cleaned:
                cur.append(cleaned)
    if cur != []:
        sentences.append(cur)
    return sentences


def align_subwords_to_words(tokens, token_embeddings, words, combine_type="mean"):
    """One sentence: sub-word tokens (strings) + their embeddings [T, D] -> one embedding per word (:254-291).
    A token equal to the current word (or '[UNK]') is that word; otherwise pieces accumulate (with the
    '##' / '▁' / 'Ġ' markers removed) until their concatenation spells the word."""
    if len(tokens) == len(words):
        return list(token_embeddings)
    out, pointer = [], 0
    word, parts = "", []
    for j, token in enumerate(tokens):
        emb = token_embeddings[j]
        current = words[pointer]
        token = token.replace("▁", "").replace("Ġ", "")
        if token == current or token == "[UNK]":
            out.append(emb)
            pointer += 1
        else:
            parts.append(emb)
            word = word + token.replace("##", "")
            if word == current:
                if combine_type == "sum":
                    merged = np.sum(np.vstack(parts), axis=0)
                elif combine_type == "mean":
                    merged = np.mean(np.vstack(parts), axis=0)
                elif combine_type == "last":
                    merged = parts[-1]
                else:
                    raise Exception("Error: not supported type to combine subword embedding.")
                out.append(merged)
                word, parts = "", []
                pointer += 1
    assert len(words) == len(out), f"==>len(sentence): {len(words)}, len(embedding): {len(out)}\ntokens:{tokens}\nsentence:{words}"
    return out


def transcript_word_features(encoder, tokenizer, sentence, lower, combine_type="mean"):
    """All word embeddings of one transcript: list of [D] arrays, in word order.  ``encoder.forward(id_lists,
    start=0, end=None, want_tokens=True)`` must return (_, tokens [sum T, D]) = sum of the last four hidden
    states of every token of the packed sentences (``BertEncoder.forward``)."""
    sentences = split_words_and_sentences(sentence, lower)
    if not sentences:
        return []
    ids = [tokenizer(s, is_split_into_words=True)["input_ids"] for s in sentences]
    _, toks = encoder.forward(ids, start=0, end=None, want_tokens=True)
    toks = toks.cpu().numpy() if hasattr(toks, "cpu") else np.asarray(toks)
    embeddings, o = [], 0
    for s, sid in zip(sentences, ids):
        n = len(sid)
        inner_ids = sid[1:n - 1]                      # skip [CLS] and [SEP] (:246-247)
        inner = toks[o + 1:o + n - 1]
        tokens = tokenizer.convert_ids_to_tokens(inner_ids)
        embeddings.extend(align_subwords_to_words(tokens, inner, s, combine_type))
        o += n
    return embeddings


def save_word_features(csv_file, embeddings, feature_level, feature_dim):
    """:296-309."""
    emb = np.array(embeddings).squeeze()
    if feature_level == "FRAME":
        if len(emb) == 0:
            emb = np.zeros((1, feature_dim))
        elif len(emb.shape) == 1:
            emb = emb[np.newaxis, :]
    else:
        if len(emb) == 0:
            emb = np.zeros((feature_dim,))
        elif len(emb.shape) == 2:
            emb = np.mean(emb, axis=0)
    if csv_file is not None:
        np.save(csv_file, emb)
    return emb


def extract_bert_embedding_english(model_name, trans_dir, save_dir, feature_level, layer_ids=None, combine_type="mean",
                                   batch_size=256, gpu=6, overwrite=False, config=None):
    """Same signature, directory naming (:181-190) and outputs as the reference; ``layer_ids`` must be the
    default last four (the fused readout of mer_bert_forward)."""
    import pandas as pd
    from transformers import AutoConfig, AutoTokenizer
    from ..encoders import BertEncoder
    from . import common
    if config is None:
        from .. import config as config  # noqa: PLW0127
    print("=" * 30 + f' Extracting "{model_name}" ' + "=" * 30)
    start_time = time.time()
    assert layer_ids is None or list(layer_ids) == [-4, -3, -2, -1], "only the last-four readout is on the H100 path"
    dir_name = f"{model_name}-4"
    save_dir = os.path.join(save_dir, dir_name + ("-FRA" if feature_level == "FRAME" else "-UTT"))
    if not os.path.exists(save_dir):
        os.makedirs(save_dir)
    elif overwrite or len(os.listdir(save_dir)) == 0:
        print(f'==> Warning: overwrite csv out dir "{dir_name}"!')
    else:
        raise Exception(f'==> Error: csv out dir "{dir_name}" already exists, set overwrite=TRUE if needed!')
    model_dir = os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"transformers/{model_name}")
    cfg = AutoConfig.from_pretrained(model_dir)
    assert cfg.model_type in ("bert", "roberta", "electra"), \
        f"only BERT/RoBERTa/ELECTRA encoders are on the H100 path, got {cfg.model_type}"
    if cfg.model_type == "electra":
        from .text import check_electra_config
        check_electra_config(cfg)  # before any weight is read
    tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    enc = BertEncoder(common.load_hf_state_dict(model_dir), device=f"cuda:{gpu}", ln_eps=cfg.layer_norm_eps,
                      position_offset=(cfg.pad_token_id + 1) if cfg.model_type == "roberta" else 0)
    lower = "uncased" in model_name or "albert" in model_name or "electra" in model_name
    df = pd.read_csv(trans_dir)
    for idx, row in df.iterrows():
        name = row["name"]
        print(f"Processing {name} ({idx}/{len(df)})...")
        emb = transcript_word_features(enc, tokenizer, row["sentence"], lower, combine_type)
        save_word_features(os.path.join(save_dir, f"{name}.npy"), emb, feature_level, enc.hidden)
    print(f"Total {len(df)} files done! Time used ({model_name}): {time.time() - start_time:.1f}s.")
