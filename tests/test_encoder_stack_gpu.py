"""Layer-by-layer float64 parity of the transformer stack (mer_run_stack, encoder.cu) in every form its callers run,
and of the readouts the encoders build on it.

Each case runs an encoder with return_hidden=True on a synthetic checkpoint and checks every layer on its own:
|hidden[l + 1] - stack_layer(hidden[l])| <= bound elementwise (tests/_kernel_refs.py), fed the GPU's own hidden[l], so
that errors do not compound down the stack.  Every case asserts the attention route it takes from the kernels a
return_hidden=False run launches (torch.profiler), and that run's readouts must equal the return_hidden=True ones bit for
bit.  Each test prints its worst |err| / bound per form.  The fp16 V^T kernel is one kernel for the "f16" and "long"
routes; at 506 .. 4096 tokens only the long-row launch can run it (mer_attention_f16_launch refuses rows over 505), so
seeing that kernel there shows the long-row launch, while the launch itself is not told apart by name.

hidden_states[0] is checked in float64 with a bound as well: the ViT patch gather (BGR -> RGB, (p / 255 - 0.5) / 0.5,
tf32), the patch GEMM with its bias and the position rows at batch stride 197, and the class row; CLIP / DINOv2 through
the generic gather on a 260 x 300 frame cropped at (17, 38) and a 224 x 224 one, patch 14 with its zero columns 588 ..
607, per-channel mean / std, the class rows and CLIP's in-place pre_layrnorm; the BERT / RoBERTa embedding LayerNorm at
768 and 1024 with position offset 0 and 2 and token ids 0 and vocab - 1.  Position and class rows are compared as the
encoder packed them (their host-side preparation, DINOv2's interpolation included, is tested in test_host_logic.py).
Frames are random in each channel, so a channel swap or a crop offset moves every patch.  The split copy the embedding
kernel writes is the operand of layer 0 in the split-bf16 form, which the layer check applies exactly.

Forms (caller: layer order, operand format, attention route by max_seqlen, FC1 activation, width):
  VitEncoder            pre-LN, fp16 (short kernel, 197) or tf32 (tf32 V^T kernel), erf, 768
  ClipVisionEncoder     pre-LN after pre_layrnorm, B/32 fp16 (tiled fp16 V^T, 50) / L/14 tf32 stack with fp16 q | k | V^T
                        (257),
                        quick-GELU, 768 / 1024
  Dinov2Encoder         pre-LN, LayerScale folded into W_o / W_fc2, as L/14 with erf, 1024
  HubertEncoder base    post-LN, fp16: 129 .. 208 the short kernel, other rows <= 505 the tiled fp16 V^T kernel,
                        506 .. 4096 the long rows, > 4096 the fallback
                        (tf32 q | k | v through attention.cu, context cast to fp16); split bf16: <= 253 tf32 V^T, then
                        fp16 V^T and the long rows, > 4096 the fallback
  HubertEncoder large   stable (pre-LN) layers run in chunks L0 + 1, 1, 1, 1 with the last hidden state LayerNormed;
                        split bf16, or fp16 up to 505 frames
  BertEncoder           post-LN, fp16 (BERT, eps 1e-12) and split bf16 (RoBERTa-large, 1024, eps 1e-5, positions + 2);
                        by sentence length, 512 tokens taking the fallback (no long rows for text)
Not covered: post-LN on tf32 operands, which no caller runs (HuBERT and BERT pass fp16 or split bf16 only); and the two
pre-LN forms for rows beyond the fp16 attention kernels (encoder.cu: attention.cu on tf32 q | k | v), which no caller in
the repository reaches at image 224: the tf32 stack's fallback, which ClipVisionEncoder takes at an image of over 505
tokens (image=336 on L/14: 577), and the fp16 stack's fallback (attention.cu + mer_cast_f16), which needs
precision="f16" forced at such an image size.  ViT has 197 tokens and HuBERT-large uses fp16 only up to 505 frames.
The hidden-state path takes equal-length HuBERT rows (mer_hubert_forward_ragged returns no hidden states), so each
HuBERT length runs as its own batch; BERT batches are ragged.  The short kernel takes rows of 129 .. 208 tokens by
default (attention_short.cu: mer_attention_short_enabled), not every row up to 249."""
import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import synthetic as S

pytestmark = pytest.mark.gpu
U = R.U32


def _assert_route(names, route):
    want = R.ATT_KERNEL[route]
    assert any(want in n for n in names), (route, names)
    others = {r: k for r, k in R.ATT_KERNEL.items() if k != want}
    assert not any(k in n for n in names for k in others.values()), (route, names)


def _layers_worst(pk, layers, mode, hidden, cu, form, final_ln=None, eps=None):
    """Worst |hidden[l + 1] - stack_layer(hidden[l])| / bound over the layers.  final_ln (stable LN): the last hidden
    state is encoder.layer_norm of the last layer's output."""
    worst = 0.0
    L = hidden.shape[0] - 1
    for l in range(L):
        w = R.packed_layer(pk, layers, l, mode)
        ref, bound = R.stack_layer(w, hidden[l], cu, form)
        if final_ln is not None and l == L - 1:
            ref, bound = R._ln_err(ref, bound, final_ln[0], final_ln[1], eps)
        r = float(((hidden[l + 1].double() - ref).abs() / bound).max())
        assert r <= 1.0, (l, r)
        worst = max(worst, r)
        del ref, bound
    return worst


def _dev(pk, ptr):
    return {t.data_ptr(): t for t in pk.tensors}[ptr].double()


def _token_sum_ratio(feats, last, n, tokens):
    x = last.double().view(n, tokens, -1)
    ref = x.sum(1)
    bound = tokens * U * x.abs().sum(1) + 1e-30
    return float(((feats.double() - ref).abs() / bound).max())


def _seq_sum(hs):
    acc = hs[0].clone()
    for h in hs[1:]:
        acc = acc + h
    return acc


def _acc_ratio(got, hs):
    """got vs the fp32 sum of hs in order; a few ulp of the sum of magnitudes."""
    bound = 4 * U * sum(h.double().abs() for h in hs) + 1e-30
    return float(((got.double() - _seq_sum(hs).double()).abs() / bound).max())


# ---- vision ----------------------------------------------------------------------------------------------------------
def _patch_hidden0(frames, y0, x0, size, p, mean, std, w, bias, pos_rest, cls_row):
    """float64 hidden_states[0] of a patch embedding before any LayerNorm, and its bound.  The gather computes
    (pix * fp32(1 / 255) - mean) / std in fp32 (2 u of |pix / 255| / std and of |a|) and stores tf32 (LAMBDA 2^-11 |a|,
    as every stored operand in stack_layer); the GEMM's products are then exact (tf32 weights), K = kpad fp32 sums,
    plus the bias and position adds of the epilogue."""
    n, dev = frames.shape[0], frames.device
    g = size // p
    f64 = lambda v: torch.tensor([float(np.float32(t)) for t in v], dtype=torch.float64, device=dev)  # noqa: E731
    pix = frames[:, y0:y0 + size, x0:x0 + size].flip(-1).double() / 255.0                  # RGB
    a = (pix - f64(mean)) / f64(std)
    ea = 2 * U * pix / f64(std) + (2 * U + R.LAMBDA * 2.0 ** -11) * a.abs()
    rows = lambda t: t.reshape(n, g, p, g, p, 3).permute(0, 1, 3, 5, 2, 4).reshape(n * g * g, 3 * p * p)  # noqa: E731
    a, ea = rows(a), rows(ea)
    assert bool((w[:, 3 * p * p:] == 0).all())
    wk = w[:, :3 * p * p]
    z = a @ wk.T + pos_rest.repeat(n, 1) + (0 if bias is None else bias)
    ez = R._lin_err(lambda t, ww: t @ ww.T, a, ea, wk, 0.0, w.shape[1]) + 2 * U * z.abs()
    D = w.shape[0]
    x = torch.cat([cls_row.expand(n, 1, D), z.view(n, g * g, D)], 1).reshape(-1, D)
    e = torch.cat([torch.zeros(n, 1, D, dtype=torch.float64, device=dev), ez.view(n, g * g, D)], 1).reshape(-1, D)
    return x, e


@pytest.mark.parametrize("precision,route", [("f16", "short"), ("tf32", "tc")])
def test_vit_stack_layers_and_readout(cuda, precision, route):
    from mertools_b200.encoders import VitEncoder
    sd = S.vit_state_dict(seed=0, layers=2)
    frames = torch.from_numpy(np.random.default_rng(5).integers(0, 256, (2, 224, 224, 3), dtype=np.uint8)).to(cuda)
    enc = VitEncoder(sd, device=cuda, precision=precision)
    feats, hidden = enc.frame_features(frames, return_hidden=True)
    feats2, names = R.attention_kernels(lambda: enc.frame_features(frames).clone())
    assert torch.equal(R.bits(feats), R.bits(feats2))
    form = R.stack_form(precision, True, 197)
    assert form["route"] == route
    _assert_route(names, route)
    hidden = hidden.reshape(3, -1, 768)
    m = enc.model
    cls = _dev(enc.pk, m.cls_pos0)
    h0, e0 = _patch_hidden0(frames, 0, 0, 224, 16, (0.5,) * 3, (0.5,) * 3, _dev(enc.pk, m.patch_w),
                            _dev(enc.pk, m.patch_b), _dev(enc.pk, m.pos_rest), cls)
    r0 = float(((hidden[0].double() - h0).abs() / (e0 + 1e-30)).max())
    assert r0 <= 1.0 and torch.equal(hidden[0].view(2, 197, 768)[:, 0].double(), cls.expand(2, 768))
    worst = _layers_worst(enc.pk, enc.layers, precision, hidden, [0, 197, 394], form)
    r = _token_sum_ratio(feats, hidden[-1], 2, 197)
    assert r <= 1.0
    print(f"ViT {precision} ({route}): hidden_states[0] {r0:.3f}; worst layer |err| / bound {worst:.3f}; "
          f"token-sum readout {r:.3f}")


@pytest.mark.parametrize("variant,route", [("b32", "f16"), ("l14", "f16"), ("dinov2", "f16")])
def test_clip_dinov2_stack_layers_and_readout(cuda, variant, route):
    """A 260 x 300 frame cropped at (17, 38) and a 224 x 224 one, through mer_clip_vision_forward; CLIP's readout
    (post_layernorm of the class rows, tf32-rounded, then the projection) in float64 with a bound, DINOv2's token sum."""
    from mertools_b200.encoders import ClipVisionEncoder, Dinov2Encoder
    if variant == "dinov2":
        enc = Dinov2Encoder(S.dinov2_state_dict(seed=17, layers=2), device=cuda)
        eps, quick, D = 1e-6, False, 1024
    else:
        enc = ClipVisionEncoder(S.clip_vision_state_dict(seed=4, variant=variant, layers=2), device=cuda)
        eps, quick, D = 1e-5, True, S.CLIP_CFGS[variant]["hidden"]
    rng = np.random.default_rng(31)
    outs = []
    for hw, (y0, x0) in (((260, 300), (17, 38)), ((224, 224), (0, 0))):
        frames = torch.from_numpy(rng.integers(0, 256, (2, hw[0], hw[1], 3), dtype=np.uint8)).to(cuda)
        emb, hidden = _clip_forward(enc, frames, y0, x0, True)
        emb2, names = R.attention_kernels(lambda: _clip_forward(enc, frames, y0, x0, False)[0])
        assert torch.equal(R.bits(emb), R.bits(emb2))
        mode = enc.precision
        T = enc.tokens
        form = R.stack_form(mode, True, T, quick=quick, eps=eps, heads=D // 64)
        assert form["route"] == route
        _assert_route(names, route)
        hidden = hidden.reshape(3, -1, D)
        m = enc.model
        cls = _dev(enc.pk, m.cls_pos0)
        h0, e0 = _patch_hidden0(frames, y0, x0, 224, enc.patch, list(m.mean), list(m.std), _dev(enc.pk, m.patch_w),
                                None, _dev(enc.pk, m.pos_rest), cls)
        assert enc.patch != 14 or m.kpad == 608
        if variant == "dinov2":
            assert torch.equal(hidden[0].view(2, T, D)[:, 0].double(), cls.expand(2, D))
        else:
            h0, e0 = R._ln_err(h0, e0, _dev(enc.pk, m.pre_ln_g), _dev(enc.pk, m.pre_ln_b), eps)
        r0 = float(((hidden[0].double() - h0).abs() / (e0 + 1e-30)).max())
        assert r0 <= 1.0
        worst = _layers_worst(enc.pk, enc.layers, mode, hidden, [0, T, 2 * T], form)
        if variant == "dinov2":
            r = _token_sum_ratio(emb, hidden[-1], 2, T)
        else:
            m = enc.model
            cls = hidden[-1].view(2, T, D)[:, 0].double()
            y, ey = R._ln_err(cls, torch.zeros_like(cls), _dev(enc.pk, m.post_ln_g), _dev(enc.pk, m.post_ln_b), eps)
            ey = ey + R.LAMBDA * R.out_rounding(y, True)
            pw = _dev(enc.pk, m.proj_w)
            ref = y @ pw.T
            bound = R._lin_err(lambda t, w: t @ w.T, y, ey, pw, 0.0, D) + U * ref.abs()
            r = float(((emb.double() - ref).abs() / bound).max())
        assert r <= 1.0
        outs.append((worst, r, r0))
    print(f"{variant} ({route}): hidden_states[0] {max(o[2] for o in outs):.3f}; worst layer |err| / bound "
          f"{max(o[0] for o in outs):.3f}; readout {max(o[1] for o in outs):.3f}")


def _clip_forward(enc, frames, y0, x0, hidden):
    """mer_clip_vision_forward on frames already at their crop geometry (the 224 x 224 window at (y0, x0))."""
    import ctypes as C

    from mertools_b200 import _lib as L
    n, H, W, _ = frames.shape
    ws = enc.ws.get(L.lib().mer_clip_vision_workspace_bytes(C.byref(enc.model), n))
    emb = torch.empty(n, enc.proj_dim, dtype=torch.float32, device=frames.device)
    hid = torch.empty(enc.n_layers + 1, n * enc.tokens, enc.hidden, dtype=torch.float32, device=frames.device) \
        if hidden else None
    L.check(enc._fwd(C.byref(enc.model), L.ptr(frames), n, H, W, y0, x0, L.ptr(ws), ws.numel(), L.ptr(emb), L.ptr(hid),
                     L.stream_ptr()))
    torch.cuda.synchronize()
    return emb, hid


# ---- audio -----------------------------------------------------------------------------------------------------------
def _wave(T, B, cuda, seed):
    n = 400 + 320 * (T - 1) + 7
    raw = torch.stack([R.speech_like(n, seed + b) for b in range(B)])
    return raw.to(cuda)


HUBERT_BASE = {"f16": [(1, "f16"), (128, "f16"), (129, "short"), (208, "short"), (209, "f16"), (249, "f16"),
                       (250, "f16"), (253, "f16"), (254, "f16"), (505, "f16"), (506, "long"), (4096, "long"),
                       (4097, "fallback")],
               "bf16x3": [(1, "tc"), (249, "tc"), (250, "tc"), (253, "tc"), (254, "f16"), (505, "f16"), (506, "long"),
                          (4096, "long"), (4097, "fallback")]}


@pytest.mark.parametrize("precision", ["f16", "bf16x3"])
def test_hubert_base_stack_layers_and_readouts(cuda, precision):
    """Post-LN layers at every route boundary; readouts: the last-four sum (MER_LN_ACC_INIT / ACC_ADD) against the fp32
    sum of hidden[-4:], the utterance mean, and with last_layer_only hidden[-1] itself."""
    from mertools_b200.encoders import HubertEncoder
    sd = S.hubert_state_dict(seed=1, layers=4)
    enc = HubertEncoder(sd, device=cuda, stack_precision=precision)
    last = HubertEncoder(sd, device=cuda, stack_precision=precision, last_layer_only=True)
    layers = enc.layers_f16 if precision == "f16" else enc.layers
    report = []
    for T, route in HUBERT_BASE[precision]:
        B = 2 if T <= 1000 else 1
        wave = _wave(T, B, cuda, 7 + T)
        assert enc.num_frames(wave.shape[1]) == T
        utt, frames, hidden = enc.forward(wave, want_frames=True, return_hidden=True)
        (utt2, frames2), names = R.attention_kernels(lambda: tuple(t.clone() for t in enc.forward(wave, want_frames=True)))
        assert torch.equal(R.bits(frames), R.bits(frames2)) and torch.equal(R.bits(utt), R.bits(utt2))
        form = R.stack_form(precision, False, T, long_rows=True, eps=1e-5)
        assert form["route"] == route
        _assert_route(names, route)
        hid = hidden.reshape(5, B * T, 768)
        worst = _layers_worst(enc.pk, layers, precision, hid, [b * T for b in range(B + 1)], form)
        r_acc = _acc_ratio(frames.reshape(-1, 768), list(hid[-4:]))
        assert r_acc <= 1.0
        mean = frames.double().mean(1)
        assert float(((utt.double() - mean).abs() / (T * U * frames.double().abs().mean(1) + 1e-30)).max()) <= 1.0
        if T <= 254:                  # the last LayerNorm initialises acc: hidden[-1] up to an ulp
            _, f_last, h_last = last.forward(wave, want_frames=True, return_hidden=True)
            assert torch.equal(R.bits(h_last), R.bits(hidden))
            assert bool(((f_last.reshape(-1, 768) - hid[-1]).abs() <= 2 * U * hid[-1].abs()).all())
        report.append(f"{T}:{route} {worst:.3f}")
        del hidden, hid, frames, frames2
    print(f"HuBERT base {precision}: worst layer |err| / bound by frames {', '.join(report)}")


@pytest.mark.parametrize("precision,lengths", [("bf16x3", [(1, "tc"), (254, "f16"), (506, "long")]),
                                               ("f16", [(208, "short"), (505, "f16"), (506, "long")])])
def test_hubert_large_stable_stack_layers_and_readouts(cuda, precision, lengths):
    """Stable (pre-LN) layers, 5 of them so that every chunk boundary of the readout loop (L0 + 1, 1, 1, 1) is crossed;
    fp16 layers apply up to 505 frames (longer clips run split bf16).  Readouts: x_{L-3} + x_{L-2} + x_{L-1} +
    LayerNorm(x_L) (hidden[-4:]) in fp32, and with last_layer_only LayerNorm(x_L) itself."""
    from mertools_b200.encoders import HubertEncoder
    sd = S.hubert_state_dict(seed=3, layers=5, large=True)
    enc = HubertEncoder(sd, device=cuda, stack_precision=precision)
    last = HubertEncoder(sd, device=cuda, stack_precision=precision, last_layer_only=True)
    fin = (_dev(enc.pk, enc.model.enc_ln_g), _dev(enc.pk, enc.model.enc_ln_b))
    report = []
    for T, route in lengths:
        mode = precision if (precision == "bf16x3" or T <= 505) else "bf16x3"
        layers = enc.layers_f16 if mode == "f16" else enc.layers
        B = 2
        wave = _wave(T, B, cuda, 11 + T)
        utt, frames, hidden = enc.forward(wave, want_frames=True, return_hidden=True)
        (utt2, frames2), names = R.attention_kernels(lambda: tuple(t.clone() for t in enc.forward(wave, want_frames=True)))
        assert torch.equal(R.bits(frames), R.bits(frames2)) and torch.equal(R.bits(utt), R.bits(utt2))
        form = R.stack_form(mode, True, T, long_rows=True, eps=1e-5, heads=16)
        assert form["route"] == route
        _assert_route(names, route)
        hid = hidden.reshape(6, B * T, 1024)
        worst = _layers_worst(enc.pk, layers, mode, hid, [b * T for b in range(B + 1)], form, final_ln=fin, eps=1e-5)
        r_acc = _acc_ratio(frames.reshape(-1, 1024), list(hid[-4:]))
        assert r_acc <= 1.0
        _, f_last, h_last = last.forward(wave, want_frames=True, return_hidden=True)
        assert torch.equal(R.bits(h_last), R.bits(hidden))
        assert torch.equal(R.bits(f_last.reshape(-1, 1024)), R.bits(hid[-1]))
        report.append(f"{T}:{mode}:{route} {worst:.3f}")
    print(f"HuBERT large {precision}: worst layer |err| / bound by frames {', '.join(report)}")


# ---- text ------------------------------------------------------------------------------------------------------------
BERT_BATCHES = [[1, 2, 63, 64, 65], [208, 129, 1], [253, 1, 64], [254, 2, 1], [512, 1]]


@pytest.mark.parametrize("model", ["bert_f16", "roberta_large_bf16x3"])
def test_bert_stack_layers_and_readout(cuda, model):
    """Ragged batches whose longest sentence sits on each side of the route boundaries, token ids 0 and vocab - 1;
    hidden_states[0] (the embedding LayerNorm) in float64 with a bound; readout: the last-four sum against the fp32 sum
    of hidden[-4:]."""
    from mertools_b200.encoders import BertEncoder
    large = model.startswith("roberta")
    vocab = 300
    sd = S.bert_state_dict(vocab, seed=2, layers=4, large=large, max_pos=514)
    eps, off, D = (1e-5, 2, 1024) if large else (1e-12, 0, 768)
    enc = BertEncoder(sd, device=cuda, ln_eps=eps, position_offset=off, precision="bf16x3" if large else "f16")
    mode = enc.precision
    layers = enc.layers_f16 if mode == "f16" else enc.layers
    rng = np.random.default_rng(13)
    report = []
    for lens in BERT_BATCHES:
        ids = [np.concatenate([[0], rng.integers(1, vocab - 1, n - 2), [vocab - 1]]) if n > 1 else np.array([vocab - 1])
               for n in lens]
        utt, toks, hidden, cu = enc.forward(ids, want_tokens=True, return_hidden=True)
        (utt2, toks2), names = R.attention_kernels(lambda: tuple(t.clone() for t in enc.forward(ids, want_tokens=True)))
        assert torch.equal(R.bits(toks), R.bits(toks2)) and torch.equal(R.bits(utt), R.bits(utt2))
        form = R.stack_form(mode, False, max(lens), eps=eps, heads=D // 64)
        _assert_route(names, form["route"])
        flat = torch.from_numpy(np.concatenate(ids)).to(cuda)
        assert int(flat.min()) == 0 and int(flat.max()) == vocab - 1
        pos = torch.from_numpy(np.concatenate([np.arange(n) for n in lens]) + off).to(cuda)
        m = enc.model
        word, ptab, ty = enc.word.double(), enc.pos.double(), _dev(enc.pk, m.type_emb0)
        v = (word[flat] + ty) + ptab[pos]
        ev = 2 * U * (word[flat].abs() + ty.abs() + ptab[pos].abs())
        h0, e0 = R._ln_err(v, ev, _dev(enc.pk, m.emb_ln_g), _dev(enc.pk, m.emb_ln_b), eps)
        r0 = float(((hidden[0].double() - h0).abs() / e0).max())
        assert r0 <= 1.0
        worst = max(r0, _layers_worst(enc.pk, layers, mode, hidden, [int(c) for c in cu], form))
        assert _acc_ratio(toks, list(hidden[-4:])) <= 1.0
        report.append(f"{max(lens)}:{form['route']} {worst:.3f}")
    print(f"{model}: worst |err| / bound (hidden_states[0] and layers) by longest sentence {', '.join(report)}")
