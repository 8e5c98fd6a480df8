"""DeBERTa / DeBERTa-v2 text branch on CPU: the orchestration (DebertaNet over TorchOps) against HF DebertaModel /
DebertaV2Model on every hidden state for each config toggle, the relative-row map against HF's own position code, the
reference golden (tests/golden/deberta_text_golden.npz, written by make_golden_deberta.py from the unmodified reference
extract_embedding), the config refusals (before any weight is read) and the C ABI refusals of
mer_disentangled_attention (fake, never-dereferenced addresses)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import deberta_text as DT
from mertools_b200.extract.ln_decoder_text import deinterleave_qkv

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4  # token-row stride of the golden's FRAME features (make_golden_deberta.py)

SMALL = dict(vocab_size=97, hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=4,
             max_position_embeddings=64, relative_attention=True, layer_norm_eps=1e-7, hidden_dropout_prob=0.0,
             attention_probs_dropout_prob=0.0)
# (family v2, config keywords): every toggle the path computes
TOGGLES = {
    "v1": (False, dict(max_relative_positions=-1, pos_att_type=["c2p", "p2c"], position_biased_input=False,
                       type_vocab_size=0)),
    "v1-short-span-positions-types": (False, dict(max_relative_positions=8, pos_att_type=["c2p", "p2c"],
                                                  position_biased_input=True, type_vocab_size=2)),
    "v2-buckets-shared-conv": (True, dict(max_relative_positions=32, position_buckets=8, norm_rel_ebd="layer_norm",
                                          share_att_key=True, pos_att_type=["p2c", "c2p"], conv_kernel_size=3,
                                          conv_act="gelu", position_biased_input=False, type_vocab_size=0)),
    "v2-unshared-positions-types": (True, dict(max_relative_positions=16, position_buckets=-1, norm_rel_ebd="none",
                                               share_att_key=False, pos_att_type=["c2p", "p2c"], conv_kernel_size=0,
                                               position_biased_input=True, type_vocab_size=2)),
}
LENS = (5, 40, 1, 23)


def hf_config(v2, kw):
    import transformers as tf
    return (tf.DebertaV2Config if v2 else tf.DebertaConfig)(**kw)


def hf_model(v2, kw, sd):
    import transformers as tf
    m = (tf.DebertaV2Model if v2 else tf.DebertaModel)(hf_config(v2, kw)).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def torch_net(v2, kw, sd, dtype=torch.float32):
    return DT.DebertaNet({k: torch.from_numpy(v) for k, v in sd.items()}, DT.TorchOps(v2, dtype=dtype),
                         DT.DebertaDims(hf_config(v2, kw)))


@pytest.mark.parametrize("name", sorted(TOGGLES))
def test_orchestration_matches_hf_on_every_hidden_state(name):
    v2, extra = TOGGLES[name]
    kw = dict(SMALL, **extra)
    sd = S.deberta_state_dict(kw, v2, seed=5)
    m = hf_model(v2, kw, sd)
    rng = np.random.default_rng(0)
    sents = [rng.integers(1, kw["vocab_size"], n) for n in LENS]
    net = torch_net(v2, kw, sd)
    with torch.no_grad():
        acc, hs = net.forward(np.concatenate(sents), list(LENS), return_hidden=True)
    assert len(hs) == kw["num_hidden_layers"] + 1
    o = 0
    for ids, n in zip(sents, LENS):
        with torch.no_grad():
            ref = m(input_ids=torch.from_numpy(ids)[None], output_hidden_states=True).hidden_states
        for k, (got, want) in enumerate(zip(hs, ref)):
            err = float((got[o:o + n] - want[0]).abs().max())
            assert err <= 5e-5, (name, n, k, err)
        err = float((acc[o:o + n] - torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]).abs().max())
        assert err <= 2e-4, (name, n, err)
        o += n


@pytest.mark.parametrize("v2,max_rel,buckets", [(False, 512, -1), (True, 512, 256), (True, 1024, 256)])
def test_rel_rows_bit_exact_against_hf_relative_positions(v2, max_rel, buckets):
    """row(d) for d in [-4095, 4095] against HF's build_relative_position plus the clamp and (v1) att_span window its
    gather applies; the 4096 x 4096 position matrix's first and last query rows cover every distance."""
    n = 4096
    x = torch.zeros(n, 1)
    if v2:
        from transformers.models.deberta_v2.modeling_deberta_v2 import build_relative_position
        rp = build_relative_position(x, x, bucket_size=buckets, max_position=max_rel)[0]
        span = buckets
        hf = torch.clamp(rp + span, 0, 2 * span - 1)
    else:
        from transformers.models.deberta.modeling_deberta import build_relative_position
        rp = build_relative_position(x, x)[0]
        att_span = min(n, max_rel)   # compute_attention_span; the gather reads the table from row max_rel - att_span
        hf = max_rel - att_span + torch.clamp(rp + att_span, 0, 2 * att_span - 1)
    # distance d = i - j: query n-1 against keys n-1 .. 0 gives 0 .. n-1, query 0 against keys n-1 .. 1 gives -(n-1) .. -1
    want = torch.cat([hf[0, 1:].flip(0), hf[n - 1].flip(0)]).to(torch.int32).numpy()
    kw = dict(SMALL, max_position_embeddings=max_rel, max_relative_positions=max_rel)
    if v2:
        kw.update(position_buckets=buckets, pos_att_type=["c2p", "p2c"])
    got = DT.rel_rows(DT.DebertaDims(hf_config(v2, kw)), n)
    assert got.dtype == np.int32 and got.shape == (2 * n - 1,)
    np.testing.assert_array_equal(got, want)


def test_deinterleave_generalises_to_head_dim_64():
    t = torch.arange(3 * 128 * 2, dtype=torch.float32).view(3 * 128, 2)
    got = deinterleave_qkv(t, 2, 64)
    for blk in range(3):
        for h in range(2):
            assert torch.equal(got[blk * 128 + h * 64:blk * 128 + (h + 1) * 64], t[h * 192 + blk * 64:h * 192 + (blk + 1) * 64])


# ---- golden -----------------------------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "deberta_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _golden_cfg(family, vocab):
    return dict(S.DEBERTA_GOLDEN_CFGS[family], vocab_size=vocab)


def test_golden_token_ids_and_offsets_match_the_tokenizer():
    import transformers
    tok = transformers.BertTokenizer(os.path.join(G, "text_vocab.txt"))
    from mertools_b200.extract.text import find_start_end_pos
    for family in ("v1", "v2"):
        g = _golden(family)
        assert (int(g["start"]), int(g["end"])) == find_start_end_pos(tok) == (1, -1)
        for i, s in enumerate(g["sentences"]):
            if not g["isnan"][i]:
                np.testing.assert_array_equal(np.array(tok(str(s))["input_ids"]), g[f"ids{i}"])


@pytest.mark.parametrize("family", ["v1", "v2"])
def test_orchestration_reproduces_the_reference_golden(family):
    g = _golden(family)
    v2 = family == "v2"
    kw = _golden_cfg(family, int(g["vocab_size"]))
    net = torch_net(v2, kw, S.deberta_state_dict(kw, v2, seed=int(g["seed"])))
    n_sent = len(g["sentences"])
    ids = [g[f"ids{i}"] for i in range(n_sent) if f"ids{i}" in g]
    with torch.no_grad():
        acc = net.forward(np.concatenate(ids), [len(x) for x in ids]).numpy()
    o, j = 0, 0
    for i in range(n_sent):
        if f"ids{i}" not in g:
            assert g["isnan"][i] and not g[f"utt{i}"].any()
            continue
        n = len(ids[j])
        if n <= 2:   # nothing left between [CLS] and [SEP]: the reference's zeros
            assert not g[f"utt{i}"].any() and not g[f"fra{i}"].any()
            o, j = o + n, j + 1
            continue
        frame = acc[o + 1:o + n - 1]
        assert int(g[f"fran{i}"]) == len(frame), (i, int(g[f"fran{i}"]), len(frame))
        want_f, want_u = g[f"fra{i}"], g[f"utt{i}"]   # the golden keeps every FRAME_STEP-th token row
        got_f = frame[::FRAME_STEP]
        assert want_f.dtype == np.float32 and want_f.shape == got_f.shape, (i, want_f.shape, got_f.shape)
        assert np.abs(got_f - want_f).max() <= 5e-5 * max(1.0, np.abs(want_f).max())
        assert np.abs(frame.mean(0) - want_u).max() <= 5e-5 * max(1.0, np.abs(want_u).max())
        o, j = o + n, j + 1


# ---- refusals ---------------------------------------------------------------------------------------------------------
class _Untouchable(dict):
    def __getitem__(self, k):
        raise AssertionError("a weight was read")

    pop = get = items = keys = values = __iter__ = __getitem__


REFUSED = {
    "relative_attention": (False, dict(relative_attention=False)),
    "pos_att_type c2p only": (False, dict(pos_att_type=["c2p"])),
    "pos_att_type p2p": (True, dict(pos_att_type=["c2p", "p2c", "p2p"])),
    "talking_head": (False, dict(talking_head=True)),
    "head size 32": (False, dict(num_attention_heads=4)),
    "embedding_size": (True, dict(embedding_size=64)),
    "hidden_act": (False, dict(hidden_act="relu")),
    "conv_act": (True, dict(conv_kernel_size=3, conv_act="tanh")),
    "conv_groups": (True, dict(conv_kernel_size=3, conv_act="gelu", conv_groups=2)),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_unsupported_configs_are_refused_before_any_weight_is_read(name):
    v2, bad = REFUSED[name]
    kw = dict(SMALL, pos_att_type=["c2p", "p2c"])
    kw.update(bad)
    cfg = hf_config(v2, kw)
    with pytest.raises(ValueError, match="DeBERTa path"):
        DT.check_deberta_config(cfg)
    with pytest.raises(ValueError, match="DeBERTa path"):
        DT.DebertaTextEncoder(_Untouchable(), cfg, device="cpu")


def test_golden_configs_are_accepted():
    for family, v2 in (("v1", False), ("v2", True)):
        DT.check_deberta_config(hf_config(v2, _golden_cfg(family, 100)))


def _cpu_lib():
    if torch.cuda.is_available():
        pytest.skip("fake device addresses are only safe where no CUDA driver can launch anything")
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return L.lib()


def _call(dll, **over):
    base = 0x7F0000000000  # never dereferenced
    a = dict(qkv=base, vt=base + (1 << 24), vt_ld=104, pos_k=base + (2 << 24), pos_q=base + (2 << 24) + 1536,
             pos_ld=1536, span=256, rel_row=base + (3 << 24), scale=0.072, ctx=base + (4 << 24),
             cu=base + (5 << 24), n_seq=2, tokens=100, max_seqlen=60, heads=12, flags=L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16)
    a.update(over)
    vp, i64 = C.c_void_p, C.c_longlong
    fn = dll.mer_disentangled_attention
    fn.restype = C.c_int
    rc = fn(vp(a["qkv"]), vp(a["vt"]), i64(a["vt_ld"]), vp(a["pos_k"]), vp(a["pos_q"]), i64(a["pos_ld"]),
            C.c_int(a["span"]), vp(a["rel_row"]), C.c_float(a["scale"]), vp(a["ctx"]), vp(a["cu"]), C.c_int(a["n_seq"]),
            i64(a["tokens"]), C.c_int(a["max_seqlen"]), C.c_int(a["heads"]), C.c_int(a["flags"]), vp(0))
    return rc, dll.mer_last_error().decode()


def test_abi_refusals_of_mer_disentangled_attention():
    dll = _cpu_lib()
    refused = {
        "heads 0": dict(heads=0), "heads 65536": dict(heads=65536),
        "vt_ld misaligned": dict(vt_ld=108), "vt_ld < tokens": dict(vt_ld=96),
        "tf32 vt_ld misaligned": dict(flags=0, vt_ld=102),
        "span 0": dict(span=0), "span negative": dict(span=-3),
        "null pos_k": dict(pos_k=None), "null pos_q": dict(pos_q=None), "null rel_row": dict(rel_row=None),
        "null qkv": dict(qkv=None),
        "pos_ld < heads * 64": dict(pos_ld=704), "pos_q misaligned": dict(pos_q=0x7F0000000000 + (2 << 24) + 8),
        "max_seqlen > tokens": dict(max_seqlen=101), "two ctx formats": dict(flags=L.MER_EPI_OUT_F16 | L.MER_EPI_SPLIT_BF16),
    }
    for name, over in refused.items():
        rc, msg = _call(dll, **over)
        assert rc != 0 and msg.startswith("mer_disentangled_attention:"), (name, rc, msg)
    # accepted arguments get past validation and stop at the first CUDA call (no driver here)
    for over in (dict(), dict(flags=L.MER_EPI_SPLIT_BF16, vt_ld=100), dict(flags=L.MER_EPI_ROUND_TF32)):
        rc, msg = _call(dll, **over)
        assert not msg.startswith("mer_disentangled_attention:"), (over, msg)
