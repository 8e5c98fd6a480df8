"""GPU parity of the BLOOM / OPT branch of the text extractor: the new kernels (causal head-dim-128 attention with ALiBi,
wide LayerNorm, the tanh-GELU and fp16 ReLU GEMM epilogues) against float64 references of the same operand values, and
the whole path — extract_embedding on the synthetic checkpoints against the golden of the unmodified reference
(1e-3, max-abs / max-ref and relative L2), a x5 stress copy under the stress-bar rule of test_bench_config_gpu.py,
packing invariance, and 3-layer stacks at the BLOOM-7B1 / OPT-13B widths against the torch restatement in fp32."""
import ctypes as C
import gzip
import os
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import ln_decoder_text as LD

pytestmark = pytest.mark.gpu
HD = 128
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENS = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 300, 2048]
NAMES = {"bloom": "bloom-7b1", "opt": "opt-13b"}
_ARGS = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int]


def _att(qkv, vt, ctx, cu, max_len, heads, slopes=None):
    args = (L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), cu.numel() - 1, qkv.shape[0], max_len, heads)
    if slopes is None:
        f = L.declare("mer_causal_attention_f16", _ARGS + [C.c_void_p])
        L.check(f(*args, L.stream_ptr()))
    else:
        f = L.declare("mer_causal_alibi_attention_f16", _ARGS + [C.c_void_p, C.c_void_p])
        L.check(f(*args, L.ptr(slopes), L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


def _ragged(lens):
    return [lens[i] for i in range(len(lens)) if i % 2 == 0] + [lens[i] for i in range(len(lens)) if i % 2 == 1]


def _att_operands(lens, heads, cuda, seed=23, pad=0, pad_value=0.0):
    g = torch.Generator(device=cuda).manual_seed(seed)
    T, D = sum(lens), heads * HD
    qkv = (torch.randn(T, 3 * D, generator=g, device=cuda) * 1.5).half()
    vt = torch.full((D, (T + 7) // 8 * 8 + pad), pad_value, dtype=torch.float16, device=cuda)
    vt[:, :T] = qkv[:, 2 * D:].T
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    return qkv, vt, cu


def _alibi_reference(qkv, cu, heads, slopes):
    """float64 causal softmax(Q K^T / sqrt(128) + slope_h * j) V (HF's form of the bias) on the device."""
    D = heads * HD
    x = qkv.double()
    out = torch.zeros(qkv.shape[0], D, dtype=torch.float64, device=qkv.device)
    sl = slopes.double()[:, None, None]
    for a, b in zip(cu.tolist()[:-1], cu.tolist()[1:]):
        n = b - a
        q, k, v = (x[a:b, i * D:(i + 1) * D].view(n, heads, HD).transpose(0, 1) for i in range(3))
        s = (q @ k.transpose(1, 2)) / HD ** 0.5 + sl * torch.arange(n, device=qkv.device, dtype=torch.float64)
        s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
        out[a:b] = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, D)
    return out


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("heads", [4, 32, 40])
def test_alibi_attention_vs_float64(cuda, heads):
    """Packed lengths 1 .. 2048 with unaligned starts; 40 heads is not a power of two (the interleaved slopes)."""
    lens = _ragged(LENS)
    qkv, vt, cu = _att_operands(lens, heads, cuda)
    slopes = LD.alibi_slopes(heads).to(cuda)
    ctx = torch.full((qkv.shape[0], heads * HD), float("nan"), dtype=torch.float16, device=cuda)
    _att(qkv, vt, ctx, cu, max(lens), heads, slopes)
    assert bool(torch.isfinite(ctx).all())
    err = _rel(ctx, _alibi_reference(qkv, cu, heads, slopes))
    print(f"ALiBi causal attention, {heads} heads: max-rel {err:.2e}")
    assert err < 2e-3, err  # fp16 P and the fp16 output rounding


def test_alibi_attention_zero_slopes_is_the_plain_kernel(cuda):
    lens, heads = _ragged(LENS), 4
    qkv, vt, cu = _att_operands(lens, heads, cuda, seed=5)
    a = _att(qkv, vt, torch.empty(sum(lens), heads * HD, dtype=torch.float16, device=cuda), cu, max(lens), heads)
    b = _att(qkv, vt, torch.empty_like(a), cu, max(lens), heads, torch.zeros(heads, device=cuda))
    assert torch.equal(a, b)


def test_alibi_attention_ignores_future_keys(cuda):
    """New K / V for positions > i of one sequence leave ctx rows <= i of it bit-identical (and the others too)."""
    lens, heads, i = [37, 300, 129], 32, 150
    qkv, vt, cu = _att_operands(lens, heads, cuda)
    slopes = LD.alibi_slopes(heads).to(cuda)
    ctx0 = _att(qkv, vt, torch.empty(sum(lens), heads * HD, dtype=torch.float16, device=cuda), cu, 300, heads, slopes)
    a = 37 + i + 1
    D = heads * HD
    qkv2, vt2 = qkv.clone(), vt.clone()
    qkv2[a:37 + 300, D:2 * D] = torch.randn(300 - i - 1, D, device=cuda).half() * 3
    vt2[:, a:37 + 300] = torch.randn(D, 300 - i - 1, device=cuda).half() * 3
    ctx1 = _att(qkv2, vt2, torch.empty_like(ctx0), cu, 300, heads, slopes)
    assert torch.equal(ctx0[:a], ctx1[:a]) and torch.equal(ctx0[37 + 300:], ctx1[37 + 300:])
    assert not torch.equal(ctx0[a:37 + 300], ctx1[a:37 + 300])


def test_alibi_attention_nan_padding_does_not_leak(cuda):
    """NaN in the V^T columns past `tokens` and in the (unread) V columns of qkv."""
    lens, heads = [5, 197, 65, 17, 131], 4
    qkv, vt, cu = _att_operands(lens, heads, cuda, pad=64, pad_value=float("nan"))
    slopes = LD.alibi_slopes(heads).to(cuda)
    ref = _alibi_reference(qkv, cu, heads, slopes)
    qkv[:, 2 * heads * HD:] = float("nan")
    ctx = _att(qkv, vt, torch.empty(sum(lens), heads * HD, dtype=torch.float16, device=cuda), cu, 197, heads, slopes)
    assert bool(torch.isfinite(ctx).all()) and _rel(ctx, ref) < 2e-3


@pytest.mark.parametrize("dim", [512, 4096, 5120])
def test_layernorm_three_output_modes(cuda, dim):
    f = L.declare("mer_layernorm_f16", [C.c_void_p] * 6 + [C.c_longlong, C.c_int, C.c_float, C.c_void_p])
    g = torch.Generator(device=cuda).manual_seed(dim)
    rows = 333
    x = torch.randn(rows, dim, generator=g, device=cuda) + 3.0   # a non-zero mean
    x[::7, ::97] = 1e3                                          # outliers
    gamma = 1 + 0.1 * torch.randn(dim, generator=g, device=cuda)
    beta = 0.1 * torch.randn(dim, generator=g, device=cuda)
    eps = 1e-5
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    ref = (xd - mu) * torch.rsqrt((xd - mu).pow(2).mean(-1, keepdim=True) + eps) * gamma.double() + beta.double()
    y16 = torch.empty(rows, dim, dtype=torch.float16, device=cuda)
    y32 = torch.empty(rows, dim, device=cuda)
    acc0 = torch.randn(rows, dim, generator=g, device=cuda)
    acc = acc0.clone()
    L.check(f(L.ptr(x), L.ptr(gamma), L.ptr(beta), L.ptr(y16), None, None, rows, dim, eps, L.stream_ptr()))
    L.check(f(L.ptr(x), L.ptr(gamma), L.ptr(beta), None, L.ptr(y32), None, rows, dim, eps, L.stream_ptr()))
    L.check(f(L.ptr(x), L.ptr(gamma), L.ptr(beta), None, None, L.ptr(acc), rows, dim, eps, L.stream_ptr()))
    both16, both32 = torch.empty_like(y16), torch.empty_like(y32)
    L.check(f(L.ptr(x), L.ptr(gamma), L.ptr(beta), L.ptr(both16), L.ptr(both32), None, rows, dim, eps, L.stream_ptr()))
    torch.cuda.synchronize()
    scale = ref.abs().max()
    assert float((y32.double() - ref).abs().max() / scale) < 1e-6
    assert (y16.double() - ref).abs().max() <= 2.0 ** -11 * scale + 1e-6      # one fp16 rounding
    assert float(((acc.double() - acc0.double()) - ref).abs().max() / scale) < 1e-6
    assert torch.equal(both16, y16) and torch.equal(both32, y32)
    assert torch.equal(y32.half(), y16)


def _bloom_gelu(x):
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))


def test_gelu_tanh_epilogue_dense_sweep(cuda):
    """|error| <= 1e-6 over [-20, 20] against torch's fp32 bloom_gelu_forward: a zero operand, the sweep as the bias."""
    N = 128 * 3125
    xs = torch.linspace(-20, 20, N, device=cuda)
    a = torch.zeros(8, 64, dtype=torch.float16, device=cuda)
    w = torch.zeros(N, 64, dtype=torch.float16, device=cuda)
    out = torch.empty(8, N, device=cuda)
    L.gemm(a, w, out, bias=xs, mode=L.MER_GEMM_F16, gelu_tanh=True)
    torch.cuda.synchronize()
    err = float((out[3] - _bloom_gelu(xs)).abs().max())
    print(f"tanh-GELU epilogue: max |error| {err:.2e} on [-20, 20] ({N} points)")
    assert err <= 1e-6 and torch.equal(out[0], out[7])


@pytest.mark.parametrize("act,f16_out", [("gelu_tanh", False), ("gelu_tanh", True), ("relu", True)])
def test_new_epilogues_with_bias_odd_rows(cuda, act, f16_out):
    g = torch.Generator(device=cuda).manual_seed(7)
    M, N, K = 333, 768, 512
    a = (torch.randn(M, K, generator=g, device=cuda)).half()
    w = (torch.randn(N, K, generator=g, device=cuda) * 0.1).half()
    bias = torch.randn(N, generator=g, device=cuda)
    out = torch.full((M, N), float("nan"), dtype=torch.float16 if f16_out else torch.float32, device=cuda)
    L.gemm(a, w, out, bias=bias, mode=L.MER_GEMM_F16, f16_out=f16_out, relu=(act == "relu"),
           gelu_tanh=(act == "gelu_tanh"))
    torch.cuda.synchronize()
    h = a.double() @ w.double().T + bias.double()
    ref = torch.relu(h) if act == "relu" else 0.5 * h * (1 + torch.tanh(0.79788456 * h * (1 + 0.044715 * h * h)))
    tol = (2.0 ** -11 if f16_out else 1e-6) * ref.abs().max() + 1e-5
    assert bool(torch.isfinite(out).all()) and float((out.double() - ref).abs().max()) <= tol


def test_new_epilogue_refusals(cuda):
    a = torch.zeros(64, 64, dtype=torch.float16, device=cuda)
    w = torch.zeros(128, 64, dtype=torch.float16, device=cuda)
    res = torch.zeros(64, 128, device=cuda)
    with pytest.raises(L.MerError, match="tanh-GELU comes alone"):
        L.gemm(a, w, torch.empty(64, 128, device=cuda), res=res, mode=L.MER_GEMM_F16, gelu_tanh=True)
    with pytest.raises(L.MerError, match="tanh-GELU comes alone"):
        L.gemm(a, w, torch.empty(64, 128, device=cuda), mode=L.MER_GEMM_F16, gelu_tanh=True, relu=True)
    with pytest.raises(L.MerError, match="fp16 output excludes"):
        L.gemm(a, w, torch.empty(64, 128, dtype=torch.float16, device=cuda), res=res, mode=L.MER_GEMM_F16,
               f16_out=True, relu=True)


# ---- end to end ------------------------------------------------------------------------------------------------------
def _config(family):
    from transformers import BloomConfig, OPTConfig
    c = S.LN_DECODER_SMALL_CFG
    if family == "bloom":
        return BloomConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], n_head=c["heads"], n_layer=c["layers"],
                           bos_token_id=0, eos_token_id=2, pad_token_id=1)
    return OPTConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], num_attention_heads=c["heads"], ffn_dim=c["ffn"],
                     num_hidden_layers=c["layers"], max_position_embeddings=c["max_pos"], word_embed_proj_dim=c["hidden"],
                     bos_token_id=2, eos_token_id=2, pad_token_id=1)


def unpack_tokenizer(family, dest):
    """The committed tokenizer fixture of ``family`` as a loadable directory (its ``*.gz`` files decompressed)."""
    src = os.path.join(G, f"{family}_tokenizer")
    os.makedirs(dest, exist_ok=True)
    for f in os.listdir(src):
        with (gzip.open if f.endswith(".gz") else open)(os.path.join(src, f), "rb") as a, \
                open(os.path.join(dest, f[:-3] if f.endswith(".gz") else f), "wb") as b:
            b.write(a.read())


def _checkpoint(root, family, scale=1.0):
    from transformers import BloomModel, OPTModel
    g = np.load(os.path.join(G, f"{family}_text_golden.npz"))
    mdir = os.path.join(root, "tools", "transformers", NAMES[family])
    cfg = _config(family)
    m = (BloomModel if family == "bloom" else OPTModel)(cfg).eval()
    sd = (S.bloom_state_dict if family == "bloom" else S.opt_state_dict)(seed=int(g["seed"]), scale=scale)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    m.save_pretrained(mdir)
    unpack_tokenizer(family, mdir)
    return g, sd, cfg, m


def _run_extract(tmp_path, g, family, level):
    import pandas as pd

    from mertools_b200.extract import text
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, "chinese": sents}).to_csv(csv, index=False)
    text.extract_embedding(NAMES[family], csv, str(tmp_path / "features"), level, gpu=0, config=cfg)
    d = tmp_path / "features" / f"{NAMES[family]}-{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("family", ["bloom", "opt"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, family, level):
    g, _, _, _ = _checkpoint(str(tmp_path), family)
    got = _run_extract(tmp_path, g, family, level)
    for i, x in enumerate(got):
        ref = g[f"{level[:3].lower()}{i}"]
        assert x.shape == ref.shape, (i, x.shape, ref.shape)
        if g["isnan"][i]:
            assert x.dtype == np.float64 and not x.any()
            continue
        assert x.dtype == np.float16, x.dtype
        m, l2 = _rel(x, ref), _rel_l2(x, ref)
        print(f"{family} {level} row {i}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (i, m, l2)


def _strip(sd, family, device=None):
    return {LD._strip(k, family): (torch.from_numpy(v).to(device).half() if device else torch.from_numpy(v))
            for k, v in sd.items()}


def _ids(g):
    return [g[f"ids{i}"] for i in range(len(g["sentences"])) if not g["isnan"][i]]


@pytest.mark.parametrize("family", ["bloom", "opt"])
def test_stress_checkpoint_x5(cuda, tmp_path, family):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|) (fp16 operands)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), family, scale=5.0)
    start = int(g["start"])
    ids = _ids(g)
    utt, _ = LD.LnDecoderTextEncoder(_strip(sd, family, cuda), cfg, device=cuda).forward(ids, start=start, end=None)
    worst, noise = 0.0, 0.0
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    m64 = LD.LnDecoderNet(_strip(sd, family), LD.TorchOps(dtype=torch.float64), fam, layers, heads, eps, max_pos)
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
    print(f"{family} x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("family", ["bloom", "opt"])
def test_sentence_alone_matches_packed(cuda, tmp_path, family):
    """Packing changes only the attention's summation order (key tiles start at the sentence's first token rounded down
    to 8 in the packed buffer; DESIGN §3), so the LLaMA bars apply: 2e-4 on the UTTERANCE feature, 5e-4 relative L2 /
    1e-3 max on the token rows."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path), family)
    enc = LD.LnDecoderTextEncoder(_strip(sd, family, cuda), cfg, device=cuda)
    start = int(g["start"])
    ids = _ids(g)
    utt_p, packed = enc.forward(ids, start=start, want_tokens=True)
    packed, utt_p = packed.cpu(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], start=start, want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j]) if len(x) - start > 0 else 0.0
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{family} sentence {j} ({len(x)} tokens): alone vs packed UTT max-rel {d_utt:.1e}, tokens rel-L2 "
              f"{d_l2:.1e}, max-rel {d_max:.1e}")
        assert d_utt <= 2e-4 and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)


def _full_width_sd(family, D, F, heads, cuda, vocab=1000, max_pos=4096):
    g = torch.Generator(device=cuda).manual_seed(17)

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=cuda) * std).half()

    def ln(p):
        return {p + ".weight": 1 + w(D, std=0.1), p + ".bias": w(D, std=0.1)}
    sd = {}
    if family == "bloom":
        sd["word_embeddings.weight"] = w(vocab, D, std=1.0)
        sd.update(ln("word_embeddings_layernorm"))
        sd.update(ln("ln_f"))
        for i in range(3):
            p = f"h.{i}."
            sd.update(ln(p + "input_layernorm"))
            sd.update(ln(p + "post_attention_layernorm"))
            sd.update({p + "self_attention.query_key_value.weight": w(3 * D, D), p + "self_attention.query_key_value.bias":
                       w(3 * D), p + "self_attention.dense.weight": w(D, D), p + "self_attention.dense.bias": w(D),
                       p + "mlp.dense_h_to_4h.weight": w(F, D), p + "mlp.dense_h_to_4h.bias": w(F),
                       p + "mlp.dense_4h_to_h.weight": w(D, F), p + "mlp.dense_4h_to_h.bias": w(D)})
    else:
        sd["embed_tokens.weight"] = w(vocab, D, std=1.0)
        sd["embed_positions.weight"] = w(max_pos + 2, D, std=0.1)
        sd.update(ln("final_layer_norm"))
        for i in range(3):
            p = f"layers.{i}."
            sd.update(ln(p + "self_attn_layer_norm"))
            sd.update(ln(p + "final_layer_norm"))
            for n in ("q", "k", "v", "out"):
                sd.update({p + f"self_attn.{n}_proj.weight": w(D, D), p + f"self_attn.{n}_proj.bias": w(D)})
            sd.update({p + "fc1.weight": w(F, D), p + "fc1.bias": w(F), p + "fc2.weight": w(D, F), p + "fc2.bias": w(D)})
    return sd


@pytest.mark.parametrize("family,D,heads,F", [("bloom", 4096, 32, 16384), ("opt", 5120, 40, 20480)])
def test_full_width_stack_matches_fp32_restatement(cuda, family, D, heads, F):
    """3 layers at the BLOOM-7B1 (4096 / 32 heads / FFN 16384) and OPT-13B (5120 / 40 / 20480) widths, random fp16
    weights: the CUDA path against the torch restatement in fp32 (TF32 off) on the same weights, under the stress-bar
    rule (err <= max(1e-3, 4 * 2^13 * |fp32 - fp64 restatement|)) and 1e-3 relative L2."""
    from transformers import BloomConfig, OPTConfig
    sd = _full_width_sd(family, D, F, heads, cuda)
    if family == "bloom":
        cfg = BloomConfig(vocab_size=1000, hidden_size=D, n_head=heads, n_layer=3)
    else:
        cfg = OPTConfig(vocab_size=1000, hidden_size=D, num_attention_heads=heads, ffn_dim=F, num_hidden_layers=3,
                        max_position_embeddings=4096, word_embed_proj_dim=D)
    fam, layers, _, _, _, eps, max_pos = LD.net_dims(cfg)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(2, 130, 12)] + [700]
    ids = [rng.integers(4, 1000, n) for n in lens]
    refs = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            ref_net = LD.LnDecoderNet(dict(sd), LD.TorchOps(cuda, dt), fam, layers, heads, eps, max_pos)
            with torch.no_grad():
                refs[dt] = ref_net.forward(np.concatenate(ids), lens).cpu()
            del ref_net
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = LD.LnDecoderTextEncoder(sd, cfg, device=cuda)
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{family} full-width stack: max-rel {m:.2e} (bar {bar:.2e}, fp32-vs-fp64 {noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < bar and l2 < 1e-3
