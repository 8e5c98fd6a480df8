"""Lexical feature extraction — H100 mirror of
MERBench/feature_extraction/text/extract_text_huggingface.py (BERT / RoBERTa / ELECTRA branch; DeBERTa / DeBERTa-v2 through
extract/deberta_text.py, XLNet through extract/xlnet_text.py and ALBERT through extract/albert_text.py, float32 like BERT; LLaMA-family decoders through extract/llama_text.py and BLOOM / OPT through
extract/ln_decoder_text.py (BLOOM / OPT / Falcon), saved as float16 like the reference's fp16 GPU run; GPT-2 through
extract/ln_decoder_text.py,
float32 like the reference's fp32 run of it).

Keeps ``extract_embedding(model_name, trans_dir, save_dir, feature_level, gpu, punc_case, language,
model_dir)`` (:139), ``find_start_end_pos`` (:90-114) and the save-dir naming (:148-157).  Token ids
come from the HF tokenizer on the host exactly as in the reference (:222, bit-exact by
construction); the batch-1 model loop (:208-231) becomes one packed variable-length device pass over
many sentences (embedding gather + LayerNorm, 12 post-LN layers, last-four sum, strip specials,
mean).
"""
from __future__ import annotations

import os
import time

import numpy as np

from ..encoders import BertEncoder
from . import common
from .packed_text import packed_token_types  # noqa: F401  (re-exported)


def find_start_end_pos(tokenizer):
    """How many special tokens wrap a sentence: probe with a 6-character Chinese sentence and look
    for the [start:end] slice that decodes back to it (reference :90-114).  BERT/RoBERTa -> (1,-1)."""
    probe = "今天天气真好"
    ids = tokenizer(probe, return_tensors="pt")["input_ids"][0]
    strip = lambda s: s.replace(" ", "")  # noqa: E731
    start = None
    for start in (0, 1, 2):
        dec = strip(tokenizer.decode(ids[start:]))
        if dec == probe:
            print(f"start: {start};  end: {None}")
            return start, None
        if dec.startswith(probe):
            break
    end = None
    for end in (-1, -2):
        if strip(tokenizer.decode(ids[start:end])) == probe:
            break
    assert strip(tokenizer.decode(ids[start:end])) == probe
    print(f"start: {start};  end: {end}")
    return start, end


class TextExtractor:
    def __init__(self, state_dict, tokenizer, device="cuda", ln_eps=1e-12, position_offset=0,
                 max_tokens_per_launch=16384, encoder=None, out_dtype=None):
        """encoder: an already built encoder with the BertEncoder ``forward`` contract (the LLaMA branch) instead of a
        BertEncoder over state_dict; out_dtype: dtype of the saved features (None: as computed, fp32)."""
        self.enc = encoder if encoder is not None else BertEncoder(state_dict, device=device, ln_eps=ln_eps,
                                                                   position_offset=position_offset)
        self.tokenizer = tokenizer
        self.start, self.end = find_start_end_pos(tokenizer)
        self.max_tokens = max_tokens_per_launch
        self.out_dtype = out_dtype

    def tokenize(self, sentence):
        return self.tokenizer(sentence, return_tensors="pt")["input_ids"][0].tolist()

    def extract_sentences(self, sentences, feature_level="UTTERANCE", save_files=None):
        """sentences: list of str (None / NaN / '' give the reference's zero vector, :236-249)."""
        import pandas as pd
        ids, where = [], []
        for i, s in enumerate(sentences):
            if s is not None and not pd.isna(s) and len(s) > 0:
                ids.append(self.tokenize(s))
                where.append(i)
        res = [[] for _ in sentences]  # [] -> the reference's zero vector (nothing to embed)
        b = 0
        while b < len(ids):
            e, tok = b, 0
            while e < len(ids) and (e == b or tok + len(ids[e]) <= self.max_tokens):
                tok += len(ids[e])
                e += 1
            utt, toks = self.enc.forward(ids[b:e], start=self.start, end=self.end,
                                         want_tokens=(feature_level == "FRAME"))
            utt = utt.cpu().numpy()
            toks = toks.cpu().numpy() if toks is not None else None
            if self.out_dtype is not None:
                utt = utt.astype(self.out_dtype)
                toks = toks.astype(self.out_dtype) if toks is not None else None
            o = 0
            for j in range(b, e):
                n = len(ids[j])
                lo, hi = (self.start or 0), n + (self.end or 0)
                if hi > lo:  # something is left after stripping the special tokens (:228-231)
                    res[where[j]] = toks[o + lo:o + hi] if feature_level == "FRAME" else utt[j - b]
                o += n
            b = e
        return [common.save_feature(save_files[i] if save_files is not None else None, r,
                                    feature_level, self.enc.hidden) for i, r in enumerate(res)]


class TokenIds(list):
    """A sentence's token ids, with the ``token_type_ids`` the tokenizer returned next to them (None if it returned
    none)."""
    token_types = None


class TokenTypeTextExtractor(TextExtractor):
    """TextExtractor whose token id lists also carry the tokenizer's token_type_ids, so that the encoder adds the
    token-type term exactly when ``model(**tokenizer(sentence))`` would: XLNet's segment term (transformers 4.x's
    XLNetTokenizer returned them, 5.x only when the tokenizer config lists them in model_input_names) and GPT-2's
    ``wte[token_type_ids]`` (BertTokenizer returns them, GPT2Tokenizer does not)."""

    def tokenize(self, sentence):
        out = self.tokenizer(sentence, return_tensors="pt")
        ids = TokenIds(out["input_ids"][0].tolist())
        if "token_type_ids" in out:
            ids.token_types = out["token_type_ids"][0].tolist()
        return ids


def _tokens_per_launch(enc, row_len):
    """Tokens per launch of a packed text encoder: what half of the device memory left after its weights holds at its
    ``bytes_per_token``, at least one sentence of ``row_len`` tokens and at most 16384."""
    import torch
    free, _ = torch.cuda.mem_get_info(enc.device)
    return int(min(16384, max(row_len, free // 2 // enc.bytes_per_token)))


def _llama_extractor(model_name, model_dir, cfg, device):
    """The reference's LLM branch (:170-175, 193-196): LlamaModel + AutoTokenizer(use_fast=False), fp16 features.
    Tokens per launch: _tokens_per_launch with a row of max_position_embeddings."""
    from transformers import AutoTokenizer

    from .llama_text import LlamaTextEncoder, check_llama_config, load_llama_weights
    check_llama_config(cfg)  # before any weight is read
    tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    enc = LlamaTextEncoder(load_llama_weights(model_dir, device, prefer_bin=(model_name == "Llama-2-13b-hf")), cfg,
                           device=device)
    tokens = _tokens_per_launch(enc, cfg.max_position_embeddings)
    return TextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens, out_dtype=np.float16)


def _ln_decoder_extractor(model_dir, cfg, device):
    """The same LLM branch for BLOOM / OPT (:170-172, 193-196) and Falcon (:188-190, 193-196): BloomModel / OPTModel /
    FalconModel + AutoTokenizer(use_fast=False), fp16 features; tokens per launch as in _llama_extractor."""
    from transformers import AutoTokenizer

    from .ln_decoder_text import LnDecoderTextEncoder, check_ln_decoder_config, load_ln_decoder_weights
    check_ln_decoder_config(cfg)  # before any weight is read
    tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    enc = LnDecoderTextEncoder(load_ln_decoder_weights(model_dir, device, cfg.model_type), cfg, device=device)
    tokens = _tokens_per_launch(enc, enc.max_pos or 2048)
    return TextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens, out_dtype=np.float16)


def _gpt2_extractor(model_name, model_dir, cfg, device):
    """The reference's GPT-2 models: wenzhong2-gpt2-chinese as GPT2Model + GPT2Tokenizer(use_fast=False) (:167-169),
    gpt2-chinese-cluecorpussmall through the AutoModel + AutoTokenizer(use_fast=False) branch (:188-190).  Neither is
    halved there, so the features are fp32.  The extractor forwards the tokenizer's token_type_ids when it returns them
    (gpt2-chinese's BertTokenizer does), as model(**inputs) does.  Tokens per launch as in _ln_decoder_extractor."""
    from .ln_decoder_text import LnDecoderTextEncoder, check_ln_decoder_config, load_ln_decoder_weights
    check_ln_decoder_config(cfg)  # before any weight is read
    tokenizer = _gpt2_tokenizer(model_name, model_dir)
    enc = LnDecoderTextEncoder(load_ln_decoder_weights(model_dir, device, "gpt2"), cfg, device=device)
    tokens = _tokens_per_launch(enc, enc.max_pos)
    return TokenTypeTextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens)


def _gpt2_tokenizer(model_name, model_dir):
    """The tokenizer the reference loads for a GPT-2 model: GPT2Tokenizer for wenzhong2-gpt2-chinese, AutoTokenizer for
    every other name (gpt2-chinese-cluecorpussmall's config names BertTokenizer), both with use_fast=False."""
    from transformers import AutoTokenizer, GPT2Tokenizer
    cls = GPT2Tokenizer if model_name == "wenzhong2-gpt2-chinese" else AutoTokenizer
    return cls.from_pretrained(model_dir, use_fast=False)


def _deberta_extractor(model_name, model_dir, cfg, device):
    """The reference's DeBERTa models (:164-166 and the AutoModel branch), fp32 features.  Tokenizer by model name as
    the reference loads it: BertTokenizer for deberta-chinese-large, AutoTokenizer(use_fast=False) otherwise.  Tokens per
    launch as in _llama_extractor."""
    from transformers import AutoTokenizer, BertTokenizer

    from .deberta_text import DebertaTextEncoder, check_deberta_config
    check_deberta_config(cfg)  # before any weight is read
    if model_name == "deberta-chinese-large":
        tokenizer = BertTokenizer.from_pretrained(model_dir, use_fast=False)
    else:
        tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    enc = DebertaTextEncoder(common.load_hf_state_dict(model_dir), cfg, device=device)
    tokens = _tokens_per_launch(enc, cfg.max_position_embeddings)
    return TextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens)


def _xlnet_extractor(model_dir, cfg, device):
    """The reference's XLNet models (the AutoModel + AutoTokenizer(use_fast=False) branch), fp32 features.  The
    extractor forwards the tokenizer's token_type_ids when it returns them, as model(**inputs) does.  Tokens per launch
    as in _deberta_extractor, with MAX_LEN (512) for the max_position_embeddings XLNet does not have."""
    from transformers import AutoTokenizer

    from .xlnet_text import MAX_LEN, XlnetTextEncoder, check_xlnet_config
    check_xlnet_config(cfg)  # before any weight is read
    tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    enc = XlnetTextEncoder(common.load_hf_state_dict(model_dir), cfg, device=device)
    tokens = _tokens_per_launch(enc, MAX_LEN)
    return TokenTypeTextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens)


def _albert_extractor(model_name, model_dir, cfg, device):
    """The reference's ALBERT models, fp32 features: albert_chinese_tiny / _small with BertTokenizer (:164-166), the
    English v2 models through the AutoModel + AutoTokenizer(use_fast=False) branch.  Tokens per launch as in
    _xlnet_extractor, with max_position_embeddings for the row length."""
    from .albert_text import AlbertTextEncoder, albert_tokenizer, check_albert_config
    check_albert_config(cfg)  # before any weight is read
    tokenizer = albert_tokenizer(model_name, model_dir)
    enc = AlbertTextEncoder(common.load_hf_state_dict(model_dir), cfg, device=device)
    tokens = _tokens_per_launch(enc, cfg.max_position_embeddings)
    return TextExtractor(None, tokenizer, encoder=enc, max_tokens_per_launch=tokens)


def check_electra_config(cfg):
    """Refuse, before any weight is read, the ELECTRA configs mer_bert_forward does not compute exactly: BERT's post-LN
    layers with erf GELU and absolute positions, heads of 64, hidden 256 / 768 / 1024, and an embedding of 128 or 256
    projected to the hidden size (or as wide as it), at least 4 layers for the last-four readout."""
    act = getattr(cfg, "hidden_act", "gelu")
    assert act == "gelu", f"ELECTRA hidden_act {act!r}: only 'gelu' (erf) is on the H100 path"
    pet = getattr(cfg, "position_embedding_type", "absolute")
    assert pet == "absolute", f"ELECTRA position_embedding_type {pet!r}: only 'absolute' is on the H100 path"
    H, heads = cfg.hidden_size, cfg.num_attention_heads
    assert H % heads == 0 and H // heads == 64, \
        f"ELECTRA num_attention_heads {heads} (hidden_size {H}): only head_dim 64 is on the H100 path"
    assert H in (256, 768, 1024), f"ELECTRA hidden_size {H}: only 256, 768 or 1024 is on the H100 path"
    E = getattr(cfg, "embedding_size", H)
    assert E in (128, 256, H), f"ELECTRA embedding_size {E}: only 128, 256 or hidden_size ({H}) is on the H100 path"
    assert cfg.intermediate_size % 128 == 0 and (E == H or 2 * E <= cfg.intermediate_size), \
        f"ELECTRA intermediate_size {cfg.intermediate_size}: a multiple of 128 (and >= 2 x embedding_size) is needed"
    assert cfg.num_hidden_layers >= 4, \
        f"ELECTRA num_hidden_layers {cfg.num_hidden_layers}: the last-four readout needs at least 4 layers"


def _electra_extractor(model_dir, cfg, device):
    """The reference's ELECTRA models (the AutoModel + AutoTokenizer(use_fast=False) branch, :188-190): ElectraModel is
    BERT's post-LN stack, behind the factorised 128-wide embedding and its projection for the small models; fp32
    features, position ids from 0, the checkpoint's LayerNorm eps."""
    from transformers import AutoTokenizer
    check_electra_config(cfg)  # before any weight is read
    tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
    return TextExtractor(common.load_hf_state_dict(model_dir), tokenizer, device=device, ln_eps=cfg.layer_norm_eps,
                         position_offset=0)


def _refuse_remote_code_falcon(model_dir):
    """AutoConfig does not know the legacy RefinedWebModel / RefinedWeb model types at all; refuse them with a message
    that says what they are, before any weight is read."""
    import json
    path = os.path.join(model_dir, "config.json")
    if os.path.exists(path):
        from .ln_decoder_text import refuse_refinedweb
        with open(path) as f:
            refuse_refinedweb(json.load(f).get("model_type"))


def extract_embedding(model_name, trans_dir, save_dir, feature_level, gpu=-1, punc_case=None,
                      language="chinese", model_dir=None, config=None, sentences_per_launch=256):
    """Same signature, naming and outputs as the reference (:139-252)."""
    import pandas as pd
    from transformers import AutoConfig, AutoTokenizer
    if config is None:
        from .. import config as config  # noqa: PLW0127
    print("=" * 30 + f' Extracting "{model_name}" ' + "=" * 30)
    start_time = time.time()
    if punc_case is None and language == "chinese" and model_dir is None:
        save_dir = os.path.join(save_dir, f"{model_name}-{feature_level[:3]}")
    elif punc_case is not None:
        save_dir = os.path.join(save_dir, f"{model_name}-punc{punc_case}-{feature_level[:3]}")
    elif language == "english":
        save_dir = os.path.join(save_dir, f"{model_name}-langeng-{feature_level[:3]}")
    elif model_dir is not None:
        prefix_name = "-".join(model_dir.split("/")[-2:])
        save_dir = os.path.join(save_dir, f"{prefix_name}-{model_name}-{feature_level[:3]}")
    os.makedirs(save_dir, exist_ok=True)
    if model_dir is None:
        model_dir = os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"transformers/{model_name}")
    assert gpu != -1, "mertools_b200 has no CPU path (reference: gpu=-1 means CPU)"
    from .. import shard
    gpu = shard.device_index(gpu)
    _refuse_remote_code_falcon(model_dir)
    cfg = AutoConfig.from_pretrained(model_dir)
    assert cfg.model_type in ("bert", "roberta", "xlm-roberta", "electra", "deberta", "deberta-v2", "xlnet", "albert",
                              "llama", "bloom", "opt", "gpt2", "falcon"), \
        f"only BERT/RoBERTa/ELECTRA/DeBERTa/XLNet/ALBERT encoders and LLaMA / BLOOM / OPT / GPT-2 / Falcon decoders are " \
        f"on the H100 path, got {cfg.model_type}"
    if cfg.model_type == "llama":
        ext = _llama_extractor(model_name, model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type in ("bloom", "opt", "falcon"):
        ext = _ln_decoder_extractor(model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type == "gpt2":
        ext = _gpt2_extractor(model_name, model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type in ("deberta", "deberta-v2"):
        ext = _deberta_extractor(model_name, model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type == "xlnet":
        ext = _xlnet_extractor(model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type == "albert":
        ext = _albert_extractor(model_name, model_dir, cfg, f"cuda:{gpu}")
    elif cfg.model_type == "electra":
        ext = _electra_extractor(model_dir, cfg, f"cuda:{gpu}")
    else:
        tokenizer = AutoTokenizer.from_pretrained(model_dir, use_fast=False)
        roberta = cfg.model_type != "bert"
        ext = TextExtractor(common.load_hf_state_dict(model_dir), tokenizer, device=f"cuda:{gpu}",
                            ln_eps=cfg.layer_norm_eps,
                            position_offset=(cfg.pad_token_id + 1) if roberta else 0)
    df = pd.read_csv(trans_dir)
    col = "chinese" if language == "chinese" else "english"
    by_name = dict(zip(df["name"], df[col]))
    # one process per GPU under torchrun: this rank's share of the rows that do not have their .npy yet
    names, rank, world = shard.my_work(list(by_name), lambda n: os.path.join(save_dir, f"{n}.npy"))
    sents = [by_name[n] for n in names]
    if world > 1:
        print(f"rank {rank}/{world}: {len(names)} sentences on cuda:{gpu}")
    for s in range(0, len(names), sentences_per_launch):
        files = [os.path.join(save_dir, f"{n}.npy") for n in names[s:s + sentences_per_launch]]
        ext.extract_sentences(sents[s:s + sentences_per_launch], feature_level, save_files=files)
    print(f"Total {len(df)} files done! Time used ({model_name}): {time.time() - start_time:.1f}s.")


def build_parser():
    """Flags of extract_text_huggingface.py:270-281."""
    import argparse
    parser = argparse.ArgumentParser(description="Run.")
    parser.add_argument("--dataset", type=str, help="input dataset")
    parser.add_argument("--gpu", type=int, default=1, help="gpu id")
    parser.add_argument("--model_name", type=str, help="name of pretrained model")
    parser.add_argument("--feature_level", type=str, default="UTTERANCE", choices=["UTTERANCE", "FRAME"], help="output types")
    parser.add_argument("--punc_case", type=str, default=None, help="test punc impact to the performance")
    parser.add_argument("--language", type=str, default="chinese", help="used language")
    parser.add_argument("--model_dir", type=str, default=None, help="used user-defined model_dir")
    return parser


def main(args, config=None):
    """Script body (:283-299): transcription CSV and save directory from config.py, then extract_embedding."""
    if config is None:
        from .. import config as config  # noqa: PLW0127
    trans_dir = config.PATH_TO_TRANSCRIPTIONS[args.dataset]
    save_dir = config.PATH_TO_FEATURES[args.dataset]
    if args.punc_case is not None:
        assert args.punc_case in ["case1", "case2", "case3"]
        trans_dir = trans_dir[:-4] + f"-{args.punc_case}.csv"
        assert os.path.exists(trans_dir)
    extract_embedding(model_name=args.model_name, trans_dir=trans_dir, save_dir=save_dir, feature_level=args.feature_level,
                      gpu=args.gpu, punc_case=args.punc_case, language=args.language, model_dir=args.model_dir, config=config)


if __name__ == "__main__":
    main(build_parser().parse_args())
