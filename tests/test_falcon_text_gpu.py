"""GPU parity of the Falcon family of the LN-decoder text branch: the new kernels (multi-query causal head-dim-64
attention, rotary embedding at head_dim 64, LayerNorm over the valid columns of padded rows) against float64
references of the same operand values, and the whole path — extract_embedding on the synthetic checkpoint against the
golden of the unmodified reference (1e-3, max-abs / max-ref and relative L2), a x5 stress copy, packing invariance, and a
3-layer stack at the Falcon-7B widths against the torch restatement in fp32."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import ln_decoder_text as LD
from mertools_b200.extract.llama_text import rope_tables

pytestmark = pytest.mark.gpu
HD = 64
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENS = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 300, 2048]
NAME = "falcon-7b"
CF = S.FALCON_SMALL_CFG
vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong


def _ragged(lens):
    return [lens[i] for i in range(len(lens)) if i % 2 == 0] + [lens[i] for i in range(len(lens)) if i % 2 == 1]


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


# ---- multi-query attention -------------------------------------------------------------------------------------------
def _mqa(qkv, ld, vt, ctx, cu, max_len, heads, tokens=None):
    f = L.declare("mer_causal_mqa_attention_f16", [vp, i64, vp, i64, vp, vp, i32, i64, i32, i32, vp])
    L.check(f(L.ptr(qkv), ld, L.ptr(vt), vt.shape[1] if vt is not None else 0, L.ptr(ctx), L.ptr(cu),
              cu.numel() - 1 if cu is not None else 0, qkv.shape[0] if tokens is None else tokens, max_len, heads,
              L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


def _mqa_operands(lens, heads, cuda, seed=23, extra=40, pad_value=0.0):
    """qkv rows of pitch (heads + 1) * 64 + extra (q | k | unread columns), V^T [64, pad8(T)]."""
    g = torch.Generator(device=cuda).manual_seed(seed)
    T = sum(lens)
    ld = (heads + 1) * HD + extra
    qkv = (torch.randn(T, ld, generator=g, device=cuda) * 1.5).half()
    v = (torch.randn(T, HD, generator=g, device=cuda) * 1.5).half()
    vt = torch.full((HD, (T + 7) // 8 * 8), pad_value, dtype=torch.float16, device=cuda)
    vt[:, :T] = v.T
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    return qkv, ld, v, vt, cu


def _mqa_reference(qkv, v, cu, heads):
    D = heads * HD
    out = torch.zeros(qkv.shape[0], D, dtype=torch.float64, device=qkv.device)
    for a, b in zip(cu.tolist()[:-1], cu.tolist()[1:]):
        n = b - a
        q = qkv[a:b, :D].double().view(n, heads, HD).transpose(0, 1)
        k = qkv[a:b, D:D + HD].double()
        s = (q @ k.T) / HD ** 0.5
        s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
        out[a:b] = (torch.softmax(s, -1) @ v[a:b].double()).transpose(0, 1).reshape(n, D)
    return out


@pytest.mark.parametrize("heads", [1, 7, 71])
def test_mqa_attention_vs_float64(cuda, heads):
    """Packed ragged lengths 1 .. 2048 (unaligned sequence starts), a row pitch wider than (heads + 1) * 64."""
    lens = _ragged(LENS)
    qkv, ld, v, vt, cu = _mqa_operands(lens, heads, cuda)
    ctx = torch.full((qkv.shape[0], heads * HD), float("nan"), dtype=torch.float16, device=cuda)
    _mqa(qkv, ld, vt, ctx, cu, max(lens), heads)
    assert bool(torch.isfinite(ctx).all())
    err = _rel(ctx, _mqa_reference(qkv, v, cu, heads))
    print(f"multi-query causal attention, {heads} heads: max-rel {err:.2e}")
    assert err < 2e-3, err  # fp16 P and the fp16 output rounding


@pytest.mark.parametrize("heads", [1, 7, 71])
def test_mqa_attention_is_the_plain_kernel_on_copied_kv(cuda, heads):
    """Bit-identical to mer_causal_attention_hd_f16(head_dim=64) with the one K / V^T head copied to every head."""
    lens = _ragged(LENS)
    qkv, ld, v, vt, cu = _mqa_operands(lens, heads, cuda, seed=5)
    T, D = qkv.shape[0], heads * HD
    full = torch.empty(T, 3 * D, dtype=torch.float16, device=cuda)
    full[:, :D] = qkv[:, :D]
    full[:, D:2 * D] = qkv[:, D:D + HD].repeat(1, heads)
    full[:, 2 * D:] = v.repeat(1, heads)
    vt_full = vt.repeat(heads, 1).contiguous()
    a = _mqa(qkv, ld, vt, torch.empty(T, D, dtype=torch.float16, device=cuda), cu, max(lens), heads)
    f = L.declare("mer_causal_attention_hd_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, vp])
    b = torch.empty_like(a)
    L.check(f(L.ptr(full), L.ptr(vt_full), vt_full.shape[1], L.ptr(b), L.ptr(cu), cu.numel() - 1, T, max(lens), heads,
              HD, L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_mqa_attention_future_and_foreign_nan_do_not_leak(cuda):
    """NaN in the keys of positions after row i of a sequence and in every key of the other sequences, and new values
    for those future positions, leave rows 0 .. i of that sequence bit-identical; NaN in the unread columns of qkv and in
    the V^T columns past `tokens` never reaches ctx.  (Values of masked keys must stay finite: their probability is an
    exact 0, and 0 * NaN is NaN.)"""
    lens, heads, i = [37, 300, 129], 7, 150
    qkv, ld, v, vt, cu = _mqa_operands(lens, heads, cuda, pad_value=float("nan"))
    T, D = qkv.shape[0], heads * HD
    qkv[:, D + HD:] = float("nan")
    ref = _mqa(qkv, ld, vt, torch.empty(T, D, dtype=torch.float16, device=cuda), cu, 300, heads)
    assert bool(torch.isfinite(ref).all())
    assert _rel(ref, _mqa_reference(qkv, v, cu, heads)) < 2e-3
    a, b = 37 + i + 1, 37 + 300
    qkv2, vt2 = qkv.clone(), vt.clone()
    qkv2[a:b, D:D + HD] = float("nan")
    qkv2[:37, D:D + HD] = float("nan")
    qkv2[b:, D:D + HD] = float("nan")
    vt2[:, a:b] = torch.randn(HD, b - a, device=cuda).half() * 3
    got = _mqa(qkv2, ld, vt2, torch.empty_like(ref), cu, 300, heads)
    assert torch.equal(got[37:a], ref[37:a])


def test_mqa_attention_refusals(cuda):
    lens, heads = [5, 9], 7
    qkv, ld, v, vt, cu = _mqa_operands(lens, heads, cuda)
    ctx = torch.empty(14, heads * HD, dtype=torch.float16, device=cuda)
    for kw, msg in [(dict(heads=0), "heads"), (dict(heads=65536), "heads"),
                    (dict(ld=(heads + 1) * HD - 8), "qkv pitch"), (dict(ld=(heads + 1) * HD + 4), "qkv pitch"),
                    (dict(vt=vt[:, :8]), "V\\^T pitch"), (dict(cu=cu[:1]), "bad grid"), (dict(ctx=None), "null"),
                    (dict(qkv=None), "null"), (dict(vt_ld=12), "V\\^T pitch")]:
        a = dict(qkv=qkv, ld=ld, vt=vt, ctx=ctx, cu=cu, heads=heads)
        a.update(kw)
        f = L.declare("mer_causal_mqa_attention_f16", [vp, i64, vp, i64, vp, vp, i32, i64, i32, i32, vp])
        vt_ld = a.pop("vt_ld", a["vt"].shape[1])
        with pytest.raises(L.MerError, match=f"mer_causal_mqa_attention_f16: .*{msg}"):
            L.check(f(L.ptr(a["qkv"]), a["ld"], L.ptr(a["vt"]), vt_ld, L.ptr(a["ctx"]), L.ptr(a["cu"]),
                      a["cu"].numel() - 1, 14, 9, a["heads"], L.stream_ptr()))


# ---- rotary at head_dim 64 -------------------------------------------------------------------------------------------
def _rope(qkv, ld, rot_heads, hd, cu, cos, sin):
    f = L.declare("mer_rope_hd_f16", [vp, i64, i64, i32, i32, vp, i32, vp, vp, vp, i32, vp])
    L.check(f(L.ptr(qkv), ld, qkv.shape[0], rot_heads, hd, L.ptr(cu), cu.numel() - 1, None, L.ptr(cos), L.ptr(sin),
              cos.shape[0], L.stream_ptr()))
    torch.cuda.synchronize()


def test_rope_head_dim_64_vs_rotate_half(cuda):
    """71 q heads + 1 k head of 64 rotated in place; the columns after them untouched."""
    heads, lens = 71, [5, 300, 1, 64]
    T, ld = sum(lens), 4736
    g = torch.Generator(device=cuda).manual_seed(3)
    qkv = (torch.randn(T, ld, generator=g, device=cuda) * 2).half()
    cos, sin = (t.to(cuda) for t in rope_tables(2048, 10000.0, HD))
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    x0 = qkv.clone()
    _rope(qkv, ld, heads + 1, HD, cu, cos, sin)
    pos = torch.cat([torch.arange(n) for n in lens]).to(cuda)
    x = x0[:, :(heads + 1) * HD].float().view(T, heads + 1, HD)
    c, s = torch.cat([cos[pos], cos[pos]], -1)[:, None], torch.cat([sin[pos], sin[pos]], -1)[:, None]
    rot = torch.cat([-x[..., HD // 2:], x[..., :HD // 2]], -1)
    ref = (x * c + rot * s).reshape(T, -1)
    got = qkv[:, :(heads + 1) * HD].float()
    assert float((got - ref).abs().max()) <= 2.0 ** -10 * float(ref.abs().max())   # one fp16 rounding
    assert torch.equal(qkv[:, (heads + 1) * HD:], x0[:, (heads + 1) * HD:])


def test_rope_hd_128_is_mer_rope_f16(cuda):
    heads, lens = 4, [7, 130, 33]
    T, ld = sum(lens), 3 * heads * 128
    g = torch.Generator(device=cuda).manual_seed(4)
    a = (torch.randn(T, ld, generator=g, device=cuda) * 2).half()
    b = a.clone()
    cos, sin = (t.to(cuda) for t in rope_tables(256, 10000.0))
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    f = L.declare("mer_rope_f16", [vp, i64, i64, i32, vp, i32, vp, vp, vp, i32, vp])
    L.check(f(L.ptr(a), ld, T, heads, L.ptr(cu), cu.numel() - 1, None, L.ptr(cos), L.ptr(sin), 256, L.stream_ptr()))
    _rope(b, ld, 2 * heads, 128, cu, cos, sin)
    assert torch.equal(a, b)
    with pytest.raises(L.MerError, match="head_dim 96"):
        _rope(b, ld, 2 * heads, 96, cu, cos, sin)


# ---- LayerNorm on padded rows ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,ld", [(448, 512), (4544, 4608)])
def test_padded_layernorm_three_output_modes(cuda, dim, ld):
    f = L.declare("mer_layernorm_ld_f16", [vp, i64, vp, vp, vp, vp, vp, i64, i32, C.c_float, vp])
    g = torch.Generator(device=cuda).manual_seed(dim)
    rows = 333
    x = torch.randn(rows, ld, generator=g, device=cuda) + 3.0
    x[::7, ::97] = 1e3
    x[:, dim:] = float("nan")                                    # pad columns are never read
    gamma = 1 + 0.1 * torch.randn(dim, generator=g, device=cuda)
    beta = 0.1 * torch.randn(dim, generator=g, device=cuda)
    eps = 1e-5
    xd = x[:, :dim].double()
    mu = xd.mean(-1, keepdim=True)
    ref = (xd - mu) * torch.rsqrt((xd - mu).pow(2).mean(-1, keepdim=True) + eps) * gamma.double() + beta.double()
    y16 = torch.full((rows, ld), 7.0, dtype=torch.float16, device=cuda)
    y32 = torch.full((rows, ld), 7.0, device=cuda)
    acc0 = torch.randn(rows, ld, generator=g, device=cuda)
    acc = acc0.clone()
    L.check(f(L.ptr(x), ld, L.ptr(gamma), L.ptr(beta), L.ptr(y16), None, None, rows, dim, eps, L.stream_ptr()))
    L.check(f(L.ptr(x), ld, L.ptr(gamma), L.ptr(beta), None, L.ptr(y32), None, rows, dim, eps, L.stream_ptr()))
    L.check(f(L.ptr(x), ld, L.ptr(gamma), L.ptr(beta), None, None, L.ptr(acc), rows, dim, eps, L.stream_ptr()))
    torch.cuda.synchronize()
    scale = ref.abs().max()
    assert float((y32[:, :dim].double() - ref).abs().max() / scale) < 1e-6
    assert (y16[:, :dim].double() - ref).abs().max() <= 2.0 ** -11 * scale + 1e-6
    assert float(((acc[:, :dim].double() - acc0[:, :dim].double()) - ref).abs().max() / scale) < 1e-6
    assert bool((y16[:, dim:] == 7).all()) and bool((y32[:, dim:] == 7).all())
    assert torch.equal(acc[:, dim:], acc0[:, dim:])
    with pytest.raises(L.MerError, match="multiple of 64"):
        L.check(f(L.ptr(x), ld, L.ptr(gamma), L.ptr(beta), L.ptr(y16), None, None, rows, dim - 32, eps, L.stream_ptr()))
    with pytest.raises(L.MerError, match="row pitch"):
        L.check(f(L.ptr(x), dim - 64, L.ptr(gamma), L.ptr(beta), L.ptr(y16), None, None, rows, dim, eps,
                  L.stream_ptr()))


# ---- end to end ------------------------------------------------------------------------------------------------------
def _config(**kw):
    from transformers import FalconConfig
    base = dict(vocab_size=CF["vocab"], hidden_size=CF["hidden"], num_attention_heads=CF["heads"],
                ffn_hidden_size=CF["ffn"], num_hidden_layers=CF["layers"], max_position_embeddings=CF["max_pos"],
                layer_norm_epsilon=1e-5, bos_token_id=0, eos_token_id=2, pad_token_id=1)
    base.update(kw)
    return FalconConfig(**base)


def _checkpoint(root, scale=1.0):
    from transformers import FalconModel
    sys.path.insert(0, G)
    try:
        from make_golden_falcon import unpack_falcon_tokenizer
    finally:
        sys.path.remove(G)
    g = np.load(os.path.join(G, "falcon_text_golden.npz"))
    mdir = os.path.join(root, "tools", "transformers", NAME)
    cfg = _config()
    m = FalconModel(cfg).eval()
    sd = S.falcon_state_dict(seed=int(g["seed"]), scale=scale)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    m.save_pretrained(mdir)
    unpack_falcon_tokenizer(mdir)
    return g, sd, cfg, m


def _run_extract(tmp_path, g, level):
    import pandas as pd

    from mertools_b200.extract import text
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, "chinese": sents}).to_csv(csv, index=False)
    text.extract_embedding(NAME, csv, str(tmp_path / "features"), level, gpu=0, config=cfg)
    d = tmp_path / "features" / f"{NAME}-{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, level):
    g, _, _, _ = _checkpoint(str(tmp_path))
    got = _run_extract(tmp_path, g, level)
    for i, x in enumerate(got):
        ref = g[f"{level[:3].lower()}{i}"]
        assert x.shape == ref.shape, (i, x.shape, ref.shape)
        if g["isnan"][i]:
            assert x.dtype == np.float64 and not x.any()
            continue
        assert x.dtype == np.float16, x.dtype
        m, l2 = _rel(x, ref), _rel_l2(x, ref)
        print(f"falcon {level} row {i}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (i, m, l2)


def _strip(sd, device=None):
    return {LD._strip(k, "falcon"): (torch.from_numpy(v).to(device).half() if device else torch.from_numpy(v))
            for k, v in sd.items()}


def _ids(g):
    return [g[f"ids{i}"] for i in range(len(g["sentences"])) if not g["isnan"][i]]


def _torch_net(sd, cfg, device, dtype):
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    return LD.LnDecoderNet(sd, LD.TorchOps(device, dtype), fam, layers, heads, eps, max_pos, theta=LD.rope_theta(cfg))


def test_stress_checkpoint_x5(cuda, tmp_path):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|) (fp16 operands)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), scale=5.0)
    start = int(g["start"])
    ids = _ids(g)
    utt, _ = LD.LnDecoderTextEncoder(_strip(sd, cuda), cfg, device=cuda).forward(ids, start=start, end=None)
    worst, noise = 0.0, 0.0
    m64 = _torch_net(_strip(sd), cfg, "cpu", torch.float64)
    with torch.no_grad():
        for j, x in enumerate(ids):
            if len(x) - start < 2:
                continue
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)[[-4, -3, -2, -1]]
            r32 = r32.sum(0)[0, start:].mean(0).numpy()
            r64 = m64.forward(x, [len(x)])[start:].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"falcon x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


def test_sentence_alone_matches_packed(cuda, tmp_path):
    """Packing changes only the attention's summation order, so the LLaMA bars apply: 2e-4 on the UTTERANCE feature,
    5e-4 relative L2 / 1e-3 max on the token rows."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path))
    enc = LD.LnDecoderTextEncoder(_strip(sd, cuda), cfg, device=cuda)
    start = int(g["start"])
    ids = _ids(g)
    utt_p, packed = enc.forward(ids, start=start, want_tokens=True)
    assert utt_p.shape[1] == packed.shape[1] == CF["hidden"]
    packed, utt_p = packed.cpu(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], start=start, want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j]) if len(x) - start > 0 else 0.0
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"falcon sentence {j} ({len(x)} tokens): alone vs packed UTT max-rel {d_utt:.1e}, tokens rel-L2 "
              f"{d_l2:.1e}, max-rel {d_max:.1e}")
        assert d_utt <= 2e-4 and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)


def test_full_width_stack_matches_fp32_restatement(cuda):
    """3 layers at the Falcon-7B widths (4544 = 71 x 64, FFN 18176), random std-0.02 fp16 weights: the CUDA path (padded
    rows of 4608, QKV N = 4736) against the torch restatement in fp32 (TF32 off) on the same weights, under the
    stress-bar rule (err <= max(1e-3, 4 * 2^13 * |fp32 - fp64 restatement|)) and 1e-3 relative L2."""
    D, heads, F, vocab = 4544, 71, 18176, 1000
    g = torch.Generator(device=cuda).manual_seed(17)

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=cuda) * std).half()
    sd = {"word_embeddings.weight": w(vocab, D, std=1.0), "ln_f.weight": 1 + w(D, std=0.1), "ln_f.bias": w(D, std=0.1)}
    for i in range(3):
        p = f"h.{i}."
        sd.update({p + "input_layernorm.weight": 1 + w(D, std=0.1), p + "input_layernorm.bias": w(D, std=0.1),
                   p + "self_attention.query_key_value.weight": w(D + 2 * HD, D),
                   p + "self_attention.dense.weight": w(D, D), p + "mlp.dense_h_to_4h.weight": w(F, D),
                   p + "mlp.dense_4h_to_h.weight": w(D, F)})
    cfg = _config(vocab_size=vocab, hidden_size=D, num_attention_heads=heads, ffn_hidden_size=F, num_hidden_layers=3)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(2, 130, 12)] + [700]
    ids = [rng.integers(4, vocab, n) for n in lens]
    refs = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            with torch.no_grad():
                refs[dt] = _torch_net(dict(sd), cfg, cuda, dt).forward(np.concatenate(ids), lens).cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = LD.LnDecoderTextEncoder(sd, cfg, device=cuda)
    _, got = enc.forward(ids, want_tokens=True)
    assert got.shape == ref.shape
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"falcon full-width stack: max-rel {m:.2e} (bar {bar:.2e}, fp32-vs-fp64 {noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < bar and l2 < 1e-3
