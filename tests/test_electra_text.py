"""CPU checks of the ELECTRA branch of the text extractor (BertEncoder over mer_bert_forward / mer_bert_forward_projected):
every config refusal of check_electra_config (before any weight is read), the key handling of an ElectraForPreTraining
checkpoint, the fp32 restatement (tests/_electra_ref.py, composed from the oracle's helpers) against HF ElectraModel /
BertModel on every hidden state and against the goldens of the unmodified reference functions (sentence level and
MER2023's English word level), the layout of MerBertEmbedProjection against its ctypes mirror, and the ABI version."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from _electra_ref import electra_features, electra_hidden_states
from mertools_b200 import synthetic as S
from mertools_b200.extract import common
from mertools_b200.extract.text import check_electra_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
FRAME_STEP = 4
FAMILIES = ("small", "base", "lert_small", "eng")
CFG_OF = {"small": "small", "base": "base", "lert_small": "lert_small", "eng": "base", "words": "base"}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _golden(family):
    g = np.load(os.path.join(G, "electra_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _kw(family, vocab):
    return dict(S.ELECTRA_GOLDEN_CFGS[CFG_OF[family]], vocab_size=vocab)


def _sd(family, g):
    kw = _kw(family, int(g["vocab_size"]))
    if family == "lert_small":
        return kw, S.electra_state_dict(dict(kw, embedding_size=kw["hidden_size"]), int(g["seed"]))
    return kw, common.normalise_hf_keys(S.electra_state_dict(kw, int(g["seed"]), pretraining=family in ("eng", "words")))


# ---- config refusals ------------------------------------------------------------------------------------------------
def _cfg(**over):
    import transformers as tf
    return tf.ElectraConfig(**dict(dict(S.ELECTRA_GOLDEN_CFGS["small"], vocab_size=100), **over))


def test_published_shapes_pass():
    import transformers as tf
    for kw in S.ELECTRA_PUBLISHED_CFGS.values():
        check_electra_config(tf.ElectraConfig(**kw))
    check_electra_config(tf.ElectraConfig())            # HF's default ElectraConfig() is ELECTRA-small


@pytest.mark.parametrize("over,field", [
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(hidden_act="relu"), "hidden_act"),
    (dict(position_embedding_type="relative_key"), "position_embedding_type"),
    (dict(num_attention_heads=8), "num_attention_heads"),              # 256 / 8 = 32
    (dict(hidden_size=384, num_attention_heads=6), "hidden_size"),      # head_dim 64, width not on the path
    (dict(hidden_size=512, num_attention_heads=8, intermediate_size=2048), "hidden_size"),
    (dict(embedding_size=64), "embedding_size"),
    (dict(embedding_size=192), "embedding_size"),
    (dict(intermediate_size=1000), "intermediate_size"),
    (dict(num_hidden_layers=3), "num_hidden_layers"),
])
def test_config_refusals_name_the_field(over, field):
    with pytest.raises(AssertionError, match=field):
        check_electra_config(_cfg(**over))


def test_extractor_refuses_before_reading_weights(tmp_path):
    """A refused config stops the ELECTRA extractor before the tokenizer or the (absent) weights would be read."""
    from mertools_b200.extract import text
    with pytest.raises(AssertionError, match="hidden_act"):
        text._electra_extractor(str(tmp_path), _cfg(hidden_act="gelu_new"), "cuda:0")


# ---- checkpoint keys ------------------------------------------------------------------------------------------------
def test_pretraining_checkpoint_keys_reduce_to_electra_model():
    import transformers as tf

    from mertools_b200.encoders import bert_model_state
    kw = dict(S.ELECTRA_GOLDEN_CFGS["small"], vocab_size=100)
    raw = S.electra_state_dict(kw, seed=1, pretraining=True)
    assert any(k.startswith("electra.") for k in raw) and any(k.startswith("discriminator_predictions.") for k in raw)
    raw["electra.embeddings.position_ids"] = np.arange(512)[None]
    sd = bert_model_state(common.normalise_hf_keys(raw))
    want = {k for k in tf.ElectraModel(tf.ElectraConfig(**kw)).state_dict() if not k.endswith(("_ids",))}
    assert set(sd) == want
    assert sd["embeddings_project.weight"].shape == (256, 128)
    assert sd["embeddings.word_embeddings.weight"].shape == (100, 128)


# ---- restatement against HF and the goldens -------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["small", "base", "lert_small"])
def test_restatement_matches_hf_on_every_hidden_state(family):
    import transformers as tf
    kw = _kw(family, 300)
    if family == "lert_small":
        bkw = {k: v for k, v in kw.items() if k != "embedding_size"}
        m = tf.BertModel(tf.BertConfig(**bkw), add_pooling_layer=False).eval()
        sd = S.electra_state_dict(dict(kw, embedding_size=kw["hidden_size"]), seed=5)
    else:
        m = tf.ElectraModel(tf.ElectraConfig(**kw)).eval()
        sd = S.electra_state_dict(kw, seed=5)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    ids = np.random.default_rng(0).integers(5, 300, 37)
    ids[0], ids[-1] = 2, 3
    with torch.no_grad():
        ref = m(torch.from_numpy(ids)[None], output_hidden_states=True).hidden_states
        got = electra_hidden_states(sd, ids, kw["num_hidden_layers"], kw["num_attention_heads"])
    assert len(got) == len(ref) == kw["num_hidden_layers"] + 1
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape and float((a - b).abs().max()) < 2e-5, (i, float((a - b).abs().max()))


@pytest.mark.parametrize("family", FAMILIES)
def test_restatement_matches_reference_golden(family):
    g = _golden(family)
    kw, sd = _sd(family, g)
    start, end = int(g["start"]), (int(g["end"]) or None)
    n = len(g["sentences"])
    with torch.no_grad():
        for i in range(n):
            if f"ids{i}" not in g or len(g[f"ids{i}"]) <= 2:
                assert not g[f"utt{i}"].any()                   # NaN / blank rows: the reference's zero vector
                continue
            for level in ("UTTERANCE", "FRAME"):
                got = electra_features(sd, g[f"ids{i}"], kw["num_hidden_layers"], kw["num_attention_heads"], start,
                                       end, level)
                ref = g[f"{level[:3].lower()}{i}"]
                if level == "FRAME":
                    assert got.shape[0] == int(g[f"fran{i}"])
                    got = got[::FRAME_STEP]
                assert got.shape == ref.shape and ref.dtype == np.float32
                assert _rel(got, ref) < 5e-5, (family, i, level, _rel(got, ref))


class _RestatedElectra:
    """The restatement behind the English word path's encoder interface (BertEncoder.forward)."""

    def __init__(self, sd, layers, heads):
        self.sd, self.layers, self.heads = sd, layers, heads

    def forward(self, id_lists, start=0, end=None, want_tokens=True):
        toks = []
        with torch.no_grad():
            for ids in id_lists:
                hs = electra_hidden_states(self.sd, ids, self.layers, self.heads)
                toks.append(torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0])
        return None, torch.cat(toks)


def test_english_word_path_restatement_matches_reference_golden():
    """MER2023's extract_bert_embedding_english lower-cases words for ELECTRA; the host logic with the restatement as
    encoder reproduces the golden of the unmodified function on an ElectraForPreTraining checkpoint."""
    import transformers as tf

    from mertools_b200.extract import text_english as TE
    g = _golden("words")
    tok = tf.BertTokenizer(os.path.join(G, "text_words_vocab.txt"), do_lower_case=True)
    kw, sd = _sd("words", g)
    enc = _RestatedElectra(sd, kw["num_hidden_layers"], kw["num_attention_heads"])
    for name, sent in zip(g["names"], g["sentences"]):
        emb = TE.transcript_word_features(enc, tok, str(sent), lower=True)
        fra = TE.save_word_features(None, emb, "FRAME", 768)
        utt = TE.save_word_features(None, emb, "UTTERANCE", 768)
        assert fra.shape == g[f"fra_{name}"].shape and _rel(fra, g[f"fra_{name}"]) < 5e-5, name
        assert utt.shape == (768,) and _rel(utt, g[f"utt_{name}"]) < 5e-5, name


def test_golden_ids_are_the_tokenizers():
    import transformers as tf
    tok = tf.BertTokenizer(os.path.join(G, "text_vocab.txt"), do_lower_case=True)
    for family in FAMILIES:
        g = _golden(family)
        for i, s in enumerate(g["sentences"]):
            if not g["isnan"][i]:
                assert tok(str(s))["input_ids"] == g[f"ids{i}"].tolist(), (family, i)


# ---- C ABI ------------------------------------------------------------------------------------------------------------
def test_projection_struct_layout_matches_the_header(tmp_path):
    from mertools_b200.encoders import MerBertEmbedProjection
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in MerBertEmbedProjection._fields_]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(
        ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "mer_b200.h")}"',
         "int main(void) {", '  printf("%zu", sizeof(MerBertEmbedProjection));']
        + [f'  printf(" %zu", offsetof(MerBertEmbedProjection, {f}));' for f in fields]
        + ['  printf("\\n");', "  return 0;", "}"]))
    subprocess.run(["gcc", "-o", str(tmp_path / "probe"), str(src)], check=True)
    want = [int(v) for v in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                           text=True).stdout.split()]
    got = [C.sizeof(MerBertEmbedProjection)] + [getattr(MerBertEmbedProjection, f).offset for f in fields]
    assert got == want


def test_abi_version_is_still_4_and_the_export_exists():
    from mertools_b200 import _lib
    dll = C.CDLL(_lib.LIB_PATH)
    assert dll.mer_abi_version() == 4
    assert hasattr(dll, "mer_bert_forward_projected") and hasattr(dll, "mer_bert_forward")
