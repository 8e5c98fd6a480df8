"""GPU parity of the GPT-2 family of the text extractor: causal attention at head_dim 64 and 96
(mer_causal_attention_hd_f16) against float64, and the whole path — extract_embedding on the synthetic checkpoints
against the goldens of the unmodified reference (tests/golden/make_golden_gpt2.py; 1e-3, max-abs / max-ref and relative
L2, float32 features), x5 stress copies under the stress-bar rule of test_bench_config_gpu.py, packing invariance, and
full-depth stacks at the gpt2-chinese-cluecorpussmall (12 x 768) and Wenzhong2.0-GPT2-3.5B (30 x 3072) shapes against
the torch restatement in fp32 and fp64."""
import ctypes as C
import gzip
import json
import os
import shutil
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import ln_decoder_text as LD

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LENS = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 300, 1024]
GOLDEN = {"gpt2-chinese-cluecorpussmall": "gpt2_chinese_text_golden.npz",
          "wenzhong2-gpt2-chinese": "wenzhong_text_golden.npz"}
NAMES = list(GOLDEN)
_ARGS = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int]


def _att_hd(qkv, vt, ctx, cu, max_len, heads, hd):
    f = L.declare("mer_causal_attention_hd_f16", _ARGS + [C.c_int, C.c_void_p])
    L.check(f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), cu.numel() - 1, qkv.shape[0], max_len, heads,
              hd, L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


def _ragged(lens):
    return [lens[i] for i in range(len(lens)) if i % 2 == 0] + [lens[i] for i in range(len(lens)) if i % 2 == 1]


def _att_operands(lens, heads, hd, cuda, seed=23, pad=0, pad_value=0.0):
    g = torch.Generator(device=cuda).manual_seed(seed)
    T, D = sum(lens), heads * hd
    qkv = (torch.randn(T, 3 * D, generator=g, device=cuda) * 1.5).half()
    vt = torch.full((D, (T + 7) // 8 * 8 + pad), pad_value, dtype=torch.float16, device=cuda)
    vt[:, :T] = qkv[:, 2 * D:].T
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    return qkv, vt, cu


def _reference(qkv, cu, heads, hd):
    """float64 causal softmax(Q K^T / sqrt(hd)) V on the device."""
    D = heads * hd
    x = qkv.double()
    out = torch.zeros(qkv.shape[0], D, dtype=torch.float64, device=qkv.device)
    for a, b in zip(cu.tolist()[:-1], cu.tolist()[1:]):
        n = b - a
        q, k, v = (x[a:b, i * D:(i + 1) * D].view(n, heads, hd).transpose(0, 1) for i in range(3))
        s = (q @ k.transpose(1, 2)) / hd ** 0.5
        s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
        out[a:b] = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, D)
    return out


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("hd,heads", [(64, 12), (96, 8)])
def test_causal_attention_vs_float64(cuda, hd, heads):
    """Packed lengths 1 .. 1024 (n_positions) with unaligned starts."""
    lens = _ragged(LENS)
    qkv, vt, cu = _att_operands(lens, heads, hd, cuda)
    ctx = torch.full((qkv.shape[0], heads * hd), float("nan"), dtype=torch.float16, device=cuda)
    _att_hd(qkv, vt, ctx, cu, max(lens), heads, hd)
    assert bool(torch.isfinite(ctx).all())
    err = _rel(ctx, _reference(qkv, cu, heads, hd))
    print(f"causal attention head_dim {hd}, {heads} heads: max-rel {err:.2e}")
    assert err < 2e-3, err  # fp16 P and the fp16 output rounding


@pytest.mark.parametrize("hd", [64, 96])
def test_causal_attention_ignores_future_keys(cuda, hd):
    """New K / V for positions > i of one sequence leave ctx rows <= i of it bit-identical (and the others too)."""
    lens, heads, i = [37, 300, 129], 8, 150
    qkv, vt, cu = _att_operands(lens, heads, hd, cuda)
    ctx0 = _att_hd(qkv, vt, torch.empty(sum(lens), heads * hd, dtype=torch.float16, device=cuda), cu, 300, heads, hd)
    a = 37 + i + 1
    D = heads * hd
    qkv2, vt2 = qkv.clone(), vt.clone()
    qkv2[a:37 + 300, D:2 * D] = torch.randn(300 - i - 1, D, device=cuda).half() * 3
    vt2[:, a:37 + 300] = torch.randn(D, 300 - i - 1, device=cuda).half() * 3
    ctx1 = _att_hd(qkv2, vt2, torch.empty_like(ctx0), cu, 300, heads, hd)
    assert torch.equal(ctx0[:a], ctx1[:a]) and torch.equal(ctx0[37 + 300:], ctx1[37 + 300:])
    assert not torch.equal(ctx0[a:37 + 300], ctx1[a:37 + 300])


@pytest.mark.parametrize("hd", [64, 96])
def test_causal_attention_nan_padding_does_not_leak(cuda, hd):
    """NaN in the V^T columns past `tokens` and in the (unread) V columns of qkv."""
    lens, heads = [5, 197, 65, 17, 131], 4
    qkv, vt, cu = _att_operands(lens, heads, hd, cuda, pad=64, pad_value=float("nan"))
    ref = _reference(qkv, cu, heads, hd)
    qkv[:, 2 * heads * hd:] = float("nan")
    ctx = _att_hd(qkv, vt, torch.empty(sum(lens), heads * hd, dtype=torch.float16, device=cuda), cu, 197, heads, hd)
    assert bool(torch.isfinite(ctx).all()) and _rel(ctx, ref) < 2e-3


def test_head_dim_128_is_the_llama_kernel(cuda):
    """mer_causal_attention_hd_f16 at 128 runs mer_causal_attention_f16's kernel: bit-identical outputs."""
    lens, heads = _ragged(LENS), 4
    qkv, vt, cu = _att_operands(lens, heads, 128, cuda, seed=5)
    a = _att_hd(qkv, vt, torch.empty(sum(lens), heads * 128, dtype=torch.float16, device=cuda), cu, max(lens), heads,
                128)
    f = L.declare("mer_causal_attention_f16", _ARGS + [C.c_void_p])
    b = torch.empty_like(a)
    L.check(f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(b), L.ptr(cu), cu.numel() - 1, qkv.shape[0], max(lens), heads,
              L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_head_dim_80_is_refused_before_any_launch(cuda):
    lens, heads, hd = [5, 70], 2, 80
    qkv, vt, cu = _att_operands(lens, heads, hd, cuda)
    ctx = torch.full((sum(lens), heads * hd), 7.0, dtype=torch.float16, device=cuda)
    f = L.declare("mer_causal_attention_hd_f16", _ARGS + [C.c_int, C.c_void_p])
    launches = L.lib().mer_launch_count
    launches.argtypes, launches.restype = [], C.c_longlong
    torch.cuda.synchronize()
    before = launches()
    rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), len(lens), sum(lens), 70, heads, hd,
           L.stream_ptr())
    torch.cuda.synchronize()
    assert rc != 0 and launches() == before
    with pytest.raises(L.MerError, match="head_dim 80"):
        L.check(rc)
    assert bool((ctx == 7.0).all())


# ---- end to end ------------------------------------------------------------------------------------------------------
def _config(name):
    from transformers import GPT2Config
    c = S.GPT2_GOLDEN_CFGS[name]
    return GPT2Config(vocab_size=c["vocab"], n_positions=c["max_pos"], n_embd=c["hidden"], n_layer=c["layers"],
                      n_head=c["heads"], n_inner=c["ffn"])


def _install_tokenizer(name, dest):
    """The committed tokenizer fixture of ``name`` (as make_golden_gpt2.install_tokenizer writes it)."""
    os.makedirs(dest, exist_ok=True)
    if name == "gpt2-chinese-cluecorpussmall":
        shutil.copyfile(os.path.join(G, "text_vocab.txt"), os.path.join(dest, "vocab.txt"))
    else:
        for f in ("vocab.json", "merges.txt"):
            with gzip.open(os.path.join(G, "opt_tokenizer", f + ".gz"), "rb") as a, open(os.path.join(dest, f), "wb") as b:
                b.write(a.read())
    with open(os.path.join(G, "gpt2_tokenizer_configs.json")) as f:
        cfg = json.load(f)[name]
    with open(os.path.join(dest, "tokenizer_config.json"), "w") as f:
        json.dump(cfg, f)


def _checkpoint(root, name, scale=1.0):
    from transformers import GPT2Model
    g = np.load(os.path.join(G, GOLDEN[name]))
    c = S.GPT2_GOLDEN_CFGS[name]
    mdir = os.path.join(root, "tools", "transformers", name)
    cfg = _config(name)
    m = GPT2Model(cfg).eval()
    sd = S.gpt2_state_dict(seed=int(g["seed"]), vocab=c["vocab"], hidden=c["hidden"], ffn=c["ffn"], layers=c["layers"],
                           max_pos=c["max_pos"], scale=scale)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    m.save_pretrained(mdir)
    _install_tokenizer(name, mdir)
    return g, sd, cfg, m


def _run_extract(tmp_path, g, name, level):
    import pandas as pd

    from mertools_b200.extract import text
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, "chinese": sents}).to_csv(csv, index=False)
    text.extract_embedding(name, csv, str(tmp_path / "features"), level, gpu=0, config=cfg)
    d = tmp_path / "features" / f"{name}-{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("name", NAMES)
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, name, level):
    g, _, _, _ = _checkpoint(str(tmp_path), name)
    got = _run_extract(tmp_path, g, name, level)
    for i, x in enumerate(got):
        ref = g[f"{level[:3].lower()}{i}"]
        assert x.shape == ref.shape, (i, x.shape, ref.shape)
        if not ref.any():   # a NaN row, or nothing left after the special tokens: the reference's zeros
            assert x.dtype == ref.dtype and not x.any()
            continue
        assert x.dtype == np.float32, x.dtype
        m, l2 = _rel(x, ref), _rel_l2(x, ref)
        print(f"{name} {level} row {i}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (i, m, l2)


def _as_loaded(sd, device=None):
    """A GPT2Model state dict as load_ln_decoder_weights names and lays it out (fp16 on ``device`` when given)."""
    out = {}
    for k, v in sd.items():
        t = torch.from_numpy(v)
        if k.endswith(LD.GPT2_CONV1D):
            t = t.T.contiguous()
        out[LD._strip(k, "gpt2")] = t.to(device).half() if device else t
    return out


def _ids_types(g):
    idx = [i for i in range(len(g["sentences"])) if not g["isnan"][i]]
    types = [g[f"types{i}"] for i in idx] if f"types{idx[0]}" in g.files else None
    return [g[f"ids{i}"] for i in idx], types


@pytest.mark.parametrize("name", NAMES)
def test_stress_checkpoint_x5(cuda, tmp_path, name):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|) (fp16 operands)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), name, scale=5.0)
    start, end = int(g["start"]), int(g["end"]) or None
    ids, tts = _ids_types(g)
    utt, _ = LD.LnDecoderTextEncoder(_as_loaded(sd, cuda), cfg, device=cuda).forward(ids, start=start, end=end,
                                                                                     token_types=tts)
    worst, noise = 0.0, 0.0
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    m64 = LD.LnDecoderNet(_as_loaded(sd), LD.TorchOps(dtype=torch.float64), fam, layers, heads, eps, max_pos)
    with torch.no_grad():
        for j, x in enumerate(ids):
            if len(x) - start + (end or 0) < 2:
                continue
            kw = dict(token_type_ids=torch.from_numpy(tts[j])[None]) if tts else {}
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True, **kw).hidden_states)
            r32 = r32[[-4, -3, -2, -1]].sum(0)[0, start:end].mean(0).numpy()
            r64 = m64.forward(x, [len(x)], token_types=tts[j] if tts else None)[start:end].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{name} x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("name", NAMES)
def test_sentence_alone_matches_packed(cuda, tmp_path, name):
    """Packing changes only the attention's summation order (key tiles start at the sentence's first token rounded down
    to 8 in the packed buffer; DESIGN §3), so the LLaMA bars apply: 2e-4 on the UTTERANCE feature, 5e-4 relative L2 /
    1e-3 max on the token rows."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path), name)
    enc = LD.LnDecoderTextEncoder(_as_loaded(sd, cuda), cfg, device=cuda)
    start, end = int(g["start"]), int(g["end"]) or None
    ids, tts = _ids_types(g)
    utt_p, packed = enc.forward(ids, start=start, end=end, want_tokens=True, token_types=tts)
    packed, utt_p = packed.cpu(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], start=start, end=end, want_tokens=True,
                                   token_types=[tts[j]] if tts else None)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j]) if len(x) - start + (end or 0) > 0 else 0.0
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{name} sentence {j} ({len(x)} tokens): alone vs packed UTT max-rel {d_utt:.1e}, tokens rel-L2 "
              f"{d_l2:.1e}, max-rel {d_max:.1e}")
        assert d_utt <= 2e-4 and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)


def _full_depth_sd(D, F, layers, cuda, vocab=1000, max_pos=1024):
    """Random fp16 GPT-2 weights as load_ln_decoder_weights lays them out ([out, in])."""
    g = torch.Generator(device=cuda).manual_seed(17)

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=cuda) * std).half()

    def ln(p):
        return {p + ".weight": 1 + w(D, std=0.1), p + ".bias": w(D, std=0.1)}
    sd = {"wte.weight": w(vocab, D, std=1.0), "wpe.weight": w(max_pos, D, std=0.1), **ln("ln_f")}
    for i in range(layers):
        p = f"h.{i}."
        sd.update({**ln(p + "ln_1"), **ln(p + "ln_2"),
                   p + "attn.c_attn.weight": w(3 * D, D), p + "attn.c_attn.bias": w(3 * D),
                   p + "attn.c_proj.weight": w(D, D), p + "attn.c_proj.bias": w(D),
                   p + "mlp.c_fc.weight": w(F, D), p + "mlp.c_fc.bias": w(F),
                   p + "mlp.c_proj.weight": w(D, F), p + "mlp.c_proj.bias": w(D)})
    return sd


@pytest.mark.parametrize("layers,D,heads,F", [(12, 768, 12, 3072), (30, 3072, 32, 12288)])
def test_full_depth_stack_matches_fp32_restatement(cuda, layers, D, heads, F):
    """Every layer at the gpt2-chinese-cluecorpussmall (12 x 768 / 12 heads / FFN 3072) and Wenzhong2.0-GPT2-3.5B
    (30 x 3072 / 32 heads / FFN 12288) shapes, random fp16 weights, a 1024-token row (n_positions) among short ones: the
    CUDA path against the torch restatement in fp32 (TF32 off) on the same weights, under the stress-bar rule
    (err <= max(1e-3, 4 * 2^13 * |fp32 - fp64 restatement|)) and 1e-3 relative L2."""
    from transformers import GPT2Config
    sd = _full_depth_sd(D, F, layers, cuda)
    cfg = GPT2Config(vocab_size=1000, n_positions=1024, n_embd=D, n_layer=layers, n_head=heads, n_inner=F)
    fam, _, _, _, _, eps, max_pos = LD.net_dims(cfg)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(2, 130, 12)] + [1024]
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
            torch.cuda.empty_cache()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = LD.LnDecoderTextEncoder(sd, cfg, device=cuda)
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    m64 = _rel(got, refs[torch.float64])
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"GPT-2 {layers} x {D} stack: max-rel {m:.2e} vs fp32 ({m64:.2e} vs fp64; bar {bar:.2e}, fp32-vs-fp64 "
          f"{noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < bar and l2 < 1e-3
