"""GPU parity of the LLaMA branch of the text extractor: the four kernels (causal head-dim-128 attention, RMSNorm,
RoPE, fp16-output SwiGLU) against float64 references of the same operand values, and the whole path —
extract_embedding on the synthetic checkpoint against the golden of the unmodified reference (1e-3, max-abs / max-ref
and relative L2), a x5 stress copy under the stress-bar rule of test_bench_config_gpu.py, packing invariance, and a
13 B-shaped layer stack against the torch restatement in fp32."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import llama_text as LT

pytestmark = pytest.mark.gpu
HD = 128
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENS = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 300, 2048]


def _fn(name, args):
    return L.declare(name, args)


def _att(qkv, vt, ctx, cu, max_len, heads):
    f = _fn("mer_causal_attention_f16", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_longlong, C.c_int, C.c_int, C.c_void_p])
    L.check(f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), cu.numel() - 1, qkv.shape[0], max_len, heads,
              L.stream_ptr()))
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


def _att_reference(qkv, cu, heads):
    """float64 causal softmax(Q K^T / sqrt(128)) V on the device."""
    D = heads * HD
    x = qkv.double()
    out = torch.zeros(qkv.shape[0], D, dtype=torch.float64, device=qkv.device)
    cu = cu.tolist()
    for a, b in zip(cu[:-1], cu[1:]):
        n = b - a
        q, k, v = (x[a:b, i * D:(i + 1) * D].view(n, heads, HD).transpose(0, 1) for i in range(3))
        s = (q @ k.transpose(1, 2)) / HD ** 0.5
        s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
        out[a:b] = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, D)
    return out


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("heads", [4, 32, 40])
def test_causal_attention_vs_float64(cuda, heads):
    lens = _ragged(LENS)
    qkv, vt, cu = _att_operands(lens, heads, cuda)
    ctx = torch.full((qkv.shape[0], heads * HD), float("nan"), dtype=torch.float16, device=cuda)
    _att(qkv, vt, ctx, cu, max(lens), heads)
    assert bool(torch.isfinite(ctx).all())
    err = _rel(ctx, _att_reference(qkv, cu, heads))
    print(f"causal attention, {heads} heads: max-rel {err:.2e}")
    assert err < 2e-3, err  # fp16 P and the fp16 output rounding


def test_causal_attention_ignores_future_keys(cuda):
    """New K / V for positions > i of one sequence leave ctx rows <= i of it bit-identical (and the others too)."""
    lens, heads, i = [37, 300, 129], 4, 150
    qkv, vt, cu = _att_operands(lens, heads, cuda)
    ctx0 = _att(qkv, vt, torch.empty(sum(lens), heads * HD, dtype=torch.float16, device=cuda), cu, 300, heads)
    a = 37 + i + 1
    D = heads * HD
    qkv2, vt2 = qkv.clone(), vt.clone()
    qkv2[a:37 + 300, D:2 * D] = torch.randn(300 - i - 1, D, device=cuda).half() * 3
    vt2[:, a:37 + 300] = torch.randn(D, 300 - i - 1, device=cuda).half() * 3
    ctx1 = _att(qkv2, vt2, torch.empty_like(ctx0), cu, 300, heads)
    assert torch.equal(ctx0[:a], ctx1[:a]) and torch.equal(ctx0[37 + 300:], ctx1[37 + 300:])
    assert not torch.equal(ctx0[a:37 + 300], ctx1[a:37 + 300])


def test_causal_attention_nan_padding_does_not_leak(cuda):
    """NaN in the V^T columns past `tokens` and in the (unread) V columns of qkv."""
    lens, heads = [5, 197, 65, 17, 131], 4
    qkv, vt, cu = _att_operands(lens, heads, cuda, pad=64, pad_value=float("nan"))
    ref = _att_reference(qkv, cu, heads)
    qkv[:, 2 * heads * HD:] = float("nan")
    ctx = _att(qkv, vt, torch.empty(sum(lens), heads * HD, dtype=torch.float16, device=cuda), cu, 197, heads)
    assert bool(torch.isfinite(ctx).all()) and _rel(ctx, ref) < 2e-3


@pytest.mark.parametrize("dim", [512, 4096, 5120])
def test_rmsnorm_both_output_modes(cuda, dim):
    f = _fn("mer_rmsnorm", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_float,
                            C.c_void_p])
    g = torch.Generator(device=cuda).manual_seed(dim)
    rows = 333
    x = torch.randn(rows, dim, generator=g, device=cuda)
    x[::7, ::97] = 1e3                                      # outliers
    w = 1 + 0.1 * torch.randn(dim, generator=g, device=cuda)
    eps = 1e-5
    xd = x.double()
    ref = w.double() * (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps))
    y = torch.empty(rows, dim, dtype=torch.float16, device=cuda)
    L.check(f(L.ptr(x), L.ptr(w), L.ptr(y), None, rows, dim, eps, L.stream_ptr()))
    acc0 = torch.randn(rows, dim, generator=g, device=cuda)
    acc = acc0.clone()
    L.check(f(L.ptr(x), L.ptr(w), None, L.ptr(acc), rows, dim, eps, L.stream_ptr()))
    torch.cuda.synchronize()
    assert (y.double() - ref).abs().max() <= 2.0 ** -11 * ref.abs().max() + 1e-6      # one fp16 rounding
    assert float(((acc.double() - acc0.double()) - ref).abs().max() / ref.abs().max()) < 1e-6


@pytest.mark.parametrize("mode", ["cu_seqlens", "positions"])
def test_rope_up_to_position_4095(cuda, mode):
    f = _fn("mer_rope_f16", [C.c_void_p, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_int, C.c_void_p])
    heads, lens = 3, [4096, 5, 300]
    T, D = sum(lens), heads * HD
    g = torch.Generator(device=cuda).manual_seed(5)
    qkv = torch.randn(T, 3 * D, generator=g, device=cuda).half()
    cos, sin = (t.to(cuda) for t in LT.rope_tables(4096, 10000.0))
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    pos = torch.cat([torch.arange(n) for n in lens]).to(torch.int32).to(cuda)
    x = qkv.double()
    out = qkv.clone()
    if mode == "cu_seqlens":
        L.check(f(L.ptr(out), 3 * D, T, heads, L.ptr(cu), len(lens), None, L.ptr(cos), L.ptr(sin), 4096, L.stream_ptr()))
    else:
        L.check(f(L.ptr(out), 3 * D, T, heads, None, 0, L.ptr(pos), L.ptr(cos), L.ptr(sin), 4096, L.stream_ptr()))
    torch.cuda.synchronize()
    c = torch.cat([cos, cos], -1)[pos.long()].double()
    s = torch.cat([sin, sin], -1)[pos.long()].double()
    for blk in range(2 * heads):
        h = x[:, blk * HD:(blk + 1) * HD]
        rot = torch.cat([-h[:, 64:], h[:, :64]], -1)
        ref = h * c + rot * s
        got = out[:, blk * HD:(blk + 1) * HD].double()
        assert float(((got - ref).abs() - 2.0 ** -11 * ref.abs()).max()) <= 1e-7, blk   # rounded once
    assert torch.equal(out[:, 2 * D:], qkv[:, 2 * D:])     # V columns untouched


def test_swiglu_f16(cuda):
    f = _fn("mer_swiglu_f16", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p])
    rows, H = 257, 1408
    x = torch.randn(rows, 2 * H, device=cuda) * 3
    out = torch.empty(rows, H, dtype=torch.float16, device=cuda)
    L.check(f(L.ptr(x), L.ptr(out), rows, H, L.stream_ptr()))
    torch.cuda.synchronize()
    xd = x.double()
    ref = torch.nn.functional.silu(xd[:, :H]) * xd[:, H:]
    assert float(((out.double() - ref).abs() - 2.0 ** -11 * ref.abs()).max()) <= 1e-6


# ---- end to end ------------------------------------------------------------------------------------------------------
def _checkpoint(root, scale=1.0):
    import shutil

    from transformers import LlamaConfig, LlamaModel
    c = S.LLAMA_SMALL_CFG
    g = np.load(os.path.join(G, "llama_text_golden.npz"))
    mdir = os.path.join(root, "tools", "transformers", "llama-7b-hf")
    cfg = LlamaConfig(vocab_size=c["vocab"], hidden_size=c["hidden"], num_attention_heads=c["heads"],
                      intermediate_size=c["ffn"], num_hidden_layers=c["layers"], max_position_embeddings=c["max_pos"],
                      rms_norm_eps=1e-6)
    m = LlamaModel(cfg)
    sd = S.llama_state_dict(seed=int(g["seed"]), scale=scale)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    m.save_pretrained(mdir)
    for f in os.listdir(os.path.join(G, "llama_tokenizer")):
        shutil.copy(os.path.join(G, "llama_tokenizer", f), mdir)
    return g, sd, cfg, m


def _run_extract(tmp_path, g, level):
    import pandas as pd

    from mertools_b200.extract import text
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, "chinese": sents}).to_csv(csv, index=False)
    text.extract_embedding("llama-7b-hf", csv, str(tmp_path / "features"), level, gpu=0, config=cfg)
    d = tmp_path / "features" / f"llama-7b-hf-{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


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
        print(f"{level} row {i}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (i, m, l2)


def _encoder(sd, cfg, cuda):
    return LT.LlamaTextEncoder({k: torch.from_numpy(v).to(cuda).half() for k, v in sd.items()}, cfg, device=cuda)


def test_stress_checkpoint_x5(cuda, tmp_path):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|) (fp16 operands)."""
    g = np.load(os.path.join(G, "llama_text_golden.npz"))
    _, sd, cfg, m = _checkpoint(str(tmp_path), scale=5.0)
    ids = [g[f"ids{i}"] for i in range(len(g["sentences"])) if not g["isnan"][i]]
    utt, _ = _encoder(sd, cfg, cuda).forward(ids, start=1, end=None)
    worst, noise = 0.0, 0.0
    m64 = LT.LlamaNet({k: torch.from_numpy(v) for k, v in sd.items()}, LT.TorchOps(dtype=torch.float64), 6, 4, 1e-6,
                      10000.0, 2048)
    with torch.no_grad():
        for j, x in enumerate(ids):
            if len(x) < 2:
                continue
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)[[-4, -3, -2, -1]]
            r32 = r32.sum(0)[0, 1:].mean(0).numpy()
            r64 = m64.forward(x, [len(x)])[1:].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"LLaMA x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


def test_sentence_alone_matches_packed(cuda, tmp_path):
    """Packing changes only the attention's summation order: a sentence's key tiles start at its first token rounded
    down to 8 in the packed buffer (sentences starting on a multiple of 8 come out bit-identical).  An fp32 difference
    that crosses an fp16 operand rounding boundary moves one element by an fp16 ulp (4.9e-4 relative) and the layers
    carry it on, so the bars are 2e-4 on the saved UTTERANCE feature, 5e-4 relative L2 / 1e-3 max on the token rows."""
    g = np.load(os.path.join(G, "llama_text_golden.npz"))
    _, sd, cfg, _ = _checkpoint(str(tmp_path))
    enc = _encoder(sd, cfg, cuda)
    ids = [g[f"ids{i}"] for i in range(len(g["sentences"])) if not g["isnan"][i]]
    utt_p, packed = enc.forward(ids, want_tokens=True)
    packed, utt_p = packed.cpu(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j]) if len(x) > 1 else 0.0
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"sentence {j} ({len(x)} tokens): alone vs packed UTT max-rel {d_utt:.1e}, tokens rel-L2 {d_l2:.1e}, "
              f"max-rel {d_max:.1e}")
        assert d_utt <= 2e-4 and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)


def test_13b_shaped_stack_matches_fp32_restatement(cuda):
    """hidden 5120, 40 heads, FFN 13824, 3 layers, random fp16 weights: the CUDA path against the torch restatement in
    fp32 (TF32 off) on the same weights, under the stress-bar rule of test_bench_config_gpu.py (fp16 operands:
    err <= max(1e-3, 4 * 2^13 * |fp32 restatement - fp64 restatement|)) and 1e-3 relative L2."""
    from transformers import LlamaConfig
    cfg = LlamaConfig(vocab_size=1000, hidden_size=5120, num_attention_heads=40, intermediate_size=13824,
                      num_hidden_layers=3, max_position_embeddings=4096, rms_norm_eps=1e-5)
    g = torch.Generator(device=cuda).manual_seed(13)
    D, I = 5120, 13824

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=cuda) * std).half()
    sd = {"embed_tokens.weight": w(1000, D, std=1.0), "norm.weight": 1 + w(D, std=0.1)}
    for i in range(3):
        p = f"layers.{i}."
        sd.update({p + f"self_attn.{n}.weight": w(D, D) for n in ("q_proj", "k_proj", "v_proj", "o_proj")})
        sd.update({p + "mlp.gate_proj.weight": w(I, D), p + "mlp.up_proj.weight": w(I, D), p + "mlp.down_proj.weight": w(D, I)})
        sd.update({p + n + ".weight": 1 + w(D, std=0.1) for n in ("input_layernorm", "post_attention_layernorm")})
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(2, 130, 12)] + [700]
    ids = [rng.integers(3, 1000, n) for n in lens]
    refs = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            ref_net = LT.LlamaNet(dict(sd), LT.TorchOps(cuda, dt), 3, 40, 1e-5, 10000.0, 4096)
            with torch.no_grad():
                refs[dt] = ref_net.forward(np.concatenate(ids), lens).cpu()
            del ref_net
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = LT.LlamaTextEncoder(sd, cfg, device=cuda)
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"13B-shaped stack: max-rel {m:.2e} (bar {bar:.2e}, fp32-vs-fp64 {noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < bar and l2 < 1e-3
