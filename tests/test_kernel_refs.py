"""CPU checks of tests/_kernel_refs.py: the float64 references the kernel-level GPU tests compare with are themselves
compared with torch's operators (or a second, independent formula) at small shapes."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _kernel_refs as R


def _g(seed):
    return torch.Generator().manual_seed(seed)


def test_layernorm_reference_is_torch_layer_norm():
    x = torch.randn(5, 512, generator=_g(0)) * 3 + 10
    g, b = torch.randn(512, generator=_g(1)), torch.randn(512, generator=_g(2))
    for eps in (1e-12, 1e-5):
        want = F.layer_norm(x.double(), (512,), g.double(), b.double(), eps)
        assert float((R.layernorm(x, g, b, eps) - want).abs().max()) < 1e-12
    # the bound separates a two-pass fp32 evaluation from the one-pass E[x^2] - E[x]^2 on a mean-10 / std-0.1 row
    x = (torch.randn(4, 768, generator=_g(3)) * 0.1 + 10).float()
    g, b = torch.ones(768), torch.zeros(768)
    ref = R.layernorm(x, g, b, 1e-5)
    bound = R.layernorm_bound(x, g, ref, 1e-5)
    mu = x.mean(-1, keepdim=True)
    two = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    one = (x - mu) / torch.sqrt((x * x).mean(-1, keepdim=True) - mu * mu + 1e-5)
    assert bool(((two.double() - ref).abs() <= bound).all())
    assert float(((one.double() - ref).abs() / bound).max()) > 3


def test_rounding_helpers():
    x = torch.tensor([1.0, 1.0 + 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -12, 3.0e38, 0.0], dtype=torch.float32)
    got = R.round_tf32_ties_away(x)
    assert got.tolist()[:4] == [1.0, 1.0 + 2.0 ** -10, -(1.0 + 2.0 ** -10), 1.0]      # ties go away from zero
    assert bool((R.bits(got) & 0x1FFF == 0).all())
    y = torch.randn(4096, generator=_g(4)) * 100
    assert torch.equal(R.round_bf16_nearest_even(y), y.bfloat16().float())
    hi, lo = y.bfloat16(), (y - y.bfloat16().float()).bfloat16()
    packed = torch.stack([hi.view(128, 32), lo.view(128, 32)], 1).reshape(1, -1).view(torch.float32)
    h2, l2 = R.split_halves(packed.view(1, 4096))
    assert torch.equal(h2[0], hi.float()) and torch.equal(l2[0], lo.float())


def test_gelu_and_swiglu_references():
    x = torch.linspace(-8, 8, 1001)
    assert float((R.gelu_erf(x) - F.gelu(x.double())).abs().max()) < 1e-14
    z = torch.randn(3, 8, generator=_g(5))
    assert float((R.swiglu(z, 4) - F.silu(z[:, :4].double()) * z[:, 4:].double()).abs().max()) < 1e-14


def test_segment_and_wave_references():
    x = torch.randn(20, 8, generator=_g(6))
    got = R.segment_reduce(x, [0, 5, 7, 9], [5, 5, 3, 20], mean=True)
    assert torch.equal(got[1], torch.zeros(8, dtype=torch.float64)) and torch.equal(got[2], got[1])
    np.testing.assert_allclose(got[3].numpy(), x[9:].double().mean(0).numpy(), rtol=1e-14)
    np.testing.assert_allclose(R.segment_reduce(x, [0], [5], mean=False)[0].numpy(), x[:5].double().sum(0).numpy(),
                               rtol=1e-14)
    w = torch.randn(2, 400, generator=_g(7)) * 1e-3 + 0.5
    want = (w.double() - w.double().mean(1, keepdim=True)) / torch.sqrt(w.double().var(1, unbiased=False, keepdim=True)
                                                                        + 1e-7)
    assert float((R.wave_normalize(w) - want).abs().max()) < 1e-10


def test_attention_references_are_scaled_dot_product_attention():
    heads, lens = 3, [1, 17, 5]
    cu = [0, 1, 18, 23]
    qkv = torch.randn(sum(lens), 3 * heads * 64, generator=_g(8))
    got, mag, _ = R.attention_packed(qkv, cu, heads)
    D = heads * 64
    for s in range(3):
        a, b = cu[s], cu[s + 1]
        q, k, v = (qkv[a:b, i * D:(i + 1) * D].double().view(b - a, heads, 64).transpose(0, 1) for i in range(3))
        want = F.scaled_dot_product_attention(q, k, v).transpose(0, 1).reshape(b - a, D)
        assert float((got[a:b] - want).abs().max()) < 1e-12
    assert bool((mag >= got.abs() - 1e-12).all())

    batch, T = 2, 9
    x = torch.randn(batch * T, 3 * D, generator=_g(9))
    bias = torch.randn(heads, T, T, generator=_g(10))
    rs = torch.randn(batch * T, heads, generator=_g(11))
    got, _, _ = R.biased_attention(x, bias, rs, batch, T, heads)
    q, k, v = (x.double().view(batch, T, 3, heads, 64)[:, :, i].transpose(1, 2) for i in range(3))
    mask = rs.double().view(batch, T, heads).permute(0, 2, 1)[..., None] * bias.double()[None]
    want = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(batch * T, D)
    assert float((got - want).abs().max()) < 1e-12

    q, k, v = (torch.randn(2, n, heads, 64, generator=_g(12 + i)) for i, n in enumerate((4, 6, 6)))
    for causal in (False, True):
        got, _, _ = R.small_attention(q, k, v, causal)
        m = None
        if causal:
            m = torch.arange(6)[None, :] <= torch.arange(4)[:, None]
        want = F.scaled_dot_product_attention(*(t.double().transpose(1, 2) for t in (q, k, v)), attn_mask=m)
        assert float((got - want.transpose(1, 2)).abs().max()) < 1e-12


def test_wavlm_gate_reference_follows_the_hf_steps():
    heads, tokens = 4, 5
    x = torch.randn(tokens, heads * 64, generator=_g(20)).double()
    w, b, c = (torch.randn(*s, generator=_g(21 + i)).double() for i, s in enumerate(((8, 64), (8,), (heads,))))
    # WavLMAttention.forward: gru_rel_pos_linear -> view(..., 2, 4).sum(-1) -> sigmoid -> chunk -> gate_a * (gate_b * c - 1) + 2
    proj = (x.view(tokens, heads, 64) @ w.T + b).view(tokens, heads, 2, 4).sum(-1)
    ga, gb = torch.sigmoid(proj).chunk(2, dim=-1)
    want = (ga * (gb * c.view(1, heads, 1) - 1.0) + 2.0)[..., 0]
    assert float((R.wavlm_gate(x, w, b, c, heads) - want).abs().max()) < 1e-14


def test_videomae_patch_layout_is_the_conv3d_unfold():
    frames = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (16, 224, 224, 3), dtype=np.uint8))
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    rows = R.videomae_patches(frames, mean, std)
    vid = (frames.flip(-1).double() / 255.0 - torch.tensor(mean, dtype=torch.float64)) / torch.tensor(
        std, dtype=torch.float64)
    vid = vid.permute(3, 0, 1, 2)[None]                                           # [1, C, T, H, W]
    w = torch.randn(2, 3, 2, 16, 16, generator=_g(30)).double()
    want = F.conv3d(vid, w, stride=(2, 16, 16)).flatten(2).transpose(1, 2)[0]     # [1568, 2]
    assert float((rows @ w.reshape(2, -1).T - want).abs().max()) < 1e-9


# ---- the fusion nets' dropout hash, float64 network and Adam ------------------------------------------------------------
HASH_PS = (0.2, 0.3, 0.5, 0.9)
HASH_N = 1 << 22          # 4M draws per statistic
HASH_SEED, HASH_W = 7, 768


def _within_5_sigma(hits, n, prob):
    sigma = math.sqrt(prob * (1.0 - prob) / n)
    return abs(hits / n - prob) <= 5 * sigma, f"{hits / n:.6f} vs {prob:.6f} (5 sigma = {5 * sigma:.1e})"


def test_keep_mask_both_seeding_forms_agree():
    """keep_hash (seed and tensor index passed apart) and fus_dropout_mask_kernel (seed + 0x1000 (m + 1) passed in) are
    the same draw; seeds past 2^63 wrap as the kernels' unsigned 64-bit arithmetic does."""
    for seed, m, step in ((7, 0, 0), (7, 3, 41), ((1 << 64) - 5, 18, 123456)):
        a = R.keep_mask(seed, m, step, 4096, 0.5)
        b = R.keep_mask((seed + 0x1000 * (m + 1)) & ((1 << 64) - 1), None, step, 4096, 0.5)
        assert a.dtype == np.bool_ and np.array_equal(a, b)
    # a hand-evaluated element: seed 0, tensor 0, step 0, i = 0 (z = 0x1000 + 0x9E37.. + 0xD1B5.. mod 2^64)
    z = (0x1000 + 0x9E3779B97F4A7C15 + 0xD1B54A32D192ED03) & ((1 << 64) - 1)
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & ((1 << 64) - 1)
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & ((1 << 64) - 1)
    z ^= z >> 31
    for p in (0.1, 0.5, 0.9):
        assert bool(R.keep_mask(0, 0, 0, 1, p)[0]) == ((z >> 40) / 2 ** 24 >= np.float32(p))


@pytest.mark.parametrize("p", HASH_PS)
def test_keep_mask_keep_rate_is_one_minus_p(p):
    q = R.keep_probability(p)
    assert q == 1.0 - math.ceil(float(np.float32(p)) * 2 ** 24) / 2 ** 24
    for seed, m, step in ((HASH_SEED, 0, 0), (HASH_SEED, 3, 41)):
        ok, msg = _within_5_sigma(int(R.keep_mask(seed, m, step, HASH_N, p).sum()), HASH_N, q)
        assert ok, f"p={p} m={m} step={step}: keep fraction {msg}"


@pytest.mark.parametrize("p", HASH_PS)
def test_keep_mask_pairs_are_uncorrelated(p):
    """Two independent keep draws agree with probability q^2 + (1 - q)^2.  A hash whose neighbouring indices, rows,
    tensors or steps were correlated (or identical) would move the fraction of equal pairs far past 5 sigma."""
    q = R.keep_probability(p)
    e = q * q + (1 - q) * (1 - q)
    base = R.keep_mask(HASH_SEED, 1, 5, HASH_N + HASH_W, p)
    pairs = {
        "neighbouring elements": (base[:HASH_N], base[1:HASH_N + 1]),
        "same column, neighbouring rows": (base[:HASH_N], base[HASH_W:HASH_N + HASH_W]),
        "tensors m, m + 1": (base[:HASH_N], R.keep_mask(HASH_SEED, 2, 5, HASH_N, p)),
        "steps s, s + 1": (base[:HASH_N], R.keep_mask(HASH_SEED, 1, 6, HASH_N, p)),
    }
    for what, (x, y) in pairs.items():
        ok, msg = _within_5_sigma(int((x == y).sum()), HASH_N, e)
        assert ok, f"p={p} {what}: equal-pair fraction {msg}"


def test_fusion_f64_matches_the_fp32_oracle_trainer():
    """fusion_f64 runs the oracle's network in float64: its losses and gradients agree with the fp32 oracle Trainer
    (same masks) to fp32 accuracy, for the utterance-level, frame-level and top-N nets."""
    from mertools_b200 import synthetic as S
    from oracle import fusion as OF
    g = _g(40)
    B, p = 5, 0.3
    cases = []
    sd = S.fusion_state_dict(seed=3, audio_dim=12, text_dim=8, video_dim=4, hidden=8, out1=3, out2=2)
    xs = [torch.randn(B, d, generator=g) for d in (12, 8, 4)]
    cases.append((sd, xs, [(torch.rand(B, d, generator=g) >= p).float() for d in (12, 8, 4, 24)]))
    sd = S.fusion_state_dict(seed=4, audio_dim=6, text_dim=5, video_dim=3, hidden=8, out1=3, out2=1,
                             feat_type="frm_align")
    xs = [torch.randn(B, T, d, generator=g) for T, d in ((3, 6), (1, 5), (4, 3))]
    cases.append((sd, xs, [(torch.rand(B, d, generator=g) >= p).float() for d in (8, 8, 8, 24)]))
    sd = S.fusion_topn_state_dict([7, 3], seed=5, hidden=8, out1=4, out2=1)
    xs = [torch.randn(B, d, generator=g) for d in (7, 3)]
    cases.append((sd, xs, [(torch.rand(B, d, generator=g) >= p).float() for d in (7, 3, 16)]))
    for sd, xs, masks in cases:
        out1 = sd["fc_out_1.weight"].shape[0]
        emo = torch.randint(0, out1, (B,), generator=g)
        val = torch.randn(B, sd["fc_out_2.weight"].shape[0], generator=g)   # [B, out2]: MSE over every element / B
        ref = R.fusion_f64(sd, xs, p, masks, emo, val)
        tr = OF.Trainer(sd, dropout=p)
        args = (xs, None, None) if "encoder0.linear_1.weight" in sd else tuple(xs)  # Attention_TOPN takes the list
        ce, mse, tot, eo, vo, grads = tr.step(*args, emo, val, masks)
        assert abs(ref["loss"][2] - tot) <= 1e-5 * max(1.0, tot) and abs(ref["loss"][0] - ce) <= 1e-5 * max(1.0, ce)
        assert float((ref["out"][1] - eo.double()).abs().max()) <= 1e-5
        for n, r in ref["grads"].items():
            assert r.dtype == torch.float64
            assert float((r - grads[n].double()).abs().max()) <= 1e-5 * max(1.0, float(r.abs().max())), n
    # the upstream form is the gradient of sum(out * w)
    sd = S.fusion_state_dict(seed=3, audio_dim=12, text_dim=8, video_dim=4, hidden=8, out1=3, out2=2)
    xs = [torch.randn(B, d, generator=g) for d in (12, 8, 4)]
    ws = [torch.randn(B, n, generator=g) for n in (8, 3, 2)]
    up = R.fusion_f64(sd, xs, upstream=ws)["up"]
    sdd = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in sd.items()}
    out = OF.attention_forward(sdd, *(x.double() for x in xs))
    sum((o * w.double()).sum() for o, w in zip(out, ws)).backward()
    for n, x in sdd.items():
        assert torch.allclose(up[n], x.grad, rtol=0, atol=1e-13), n


def test_adam_f64_is_torch_adam_after_clip_grad_value():
    g = _g(41)
    p0 = torch.randn(257, generator=g, dtype=torch.float64)
    hp = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5)
    for clip, scale in ((0.0, 1.0), (0.01, 1.0), (0.0, 0.5)):
        w = p0.clone().requires_grad_(True)
        # hyper-parameters already at fp32 values, so that adam_f64's rounding of them to fp32 changes nothing
        hp32 = dict(lr=float(np.float32(1e-3)), betas=(float(np.float32(0.9)), float(np.float32(0.999))),
                    eps=float(np.float32(1e-8)), weight_decay=float(np.float32(1e-5)))
        opt = torch.optim.Adam([w], **hp32)
        p, m, v = p0.clone(), torch.zeros(257, dtype=torch.float64), torch.zeros(257, dtype=torch.float64)
        for t in range(1, 6):
            grad = torch.randn(257, generator=g, dtype=torch.float64) * 0.05
            w.grad = grad * scale
            if clip > 0:
                torch.nn.utils.clip_grad_value_([w], float(np.float32(clip)))  # the kernels take the fp32 value
            opt.step()
            p, m, v = R.adam_f64(p, grad, m, v, t, hp["lr"], *hp["betas"], hp["eps"], hp["weight_decay"],
                                 grad_scale=scale, clip=clip)
            st = opt.state[w]
            # torch moves exp_avg by lerp (m + (1 - beta1) (g - m)): the two forms differ by float64 roundings only
            for mine, theirs in ((p, w.detach()), (m, st["exp_avg"]), (v, st["exp_avg_sq"])):
                assert float((mine - theirs).abs().max()) <= 1e-14 * float(theirs.abs().max())


# ---- HuBERT conv0 ------------------------------------------------------------------------------------------------------
def _normalised(x):
    return R.wave_normalize(x[None]).float()


@pytest.mark.parametrize("frames", [1, 2, 1024, 1025, 15999])
def test_conv0_statistics_from_tap_moments_are_group_norms(frames):
    """The identity the GroupNorm statistics kernels rest on: per channel, the mean and biased variance of conv0 over a
    clip follow from the 10 tap sums and the 55 tap products of the waveform, so the normalised output equals
    F.group_norm's (num_groups = channels) in float64 -- on a normalised clip and on one with a DC offset 100x its
    noise.  Three samples past the last window make no frame and must not count."""
    w0, _, _, _ = R.conv0_weights(0)
    n = 5 * (frames - 1) + 10 + 3
    for x in (_normalised(R.speech_like(n, 1)), R.speech_like(n, 2, dc=30.0)[None]):
        y, _ = R.conv0(x, w0)
        assert y.shape[1] == frames
        X, Rm = R.conv0_moments(x, frames)
        mean, var = R.conv0_stats_from_moments(X, Rm, w0, frames)
        var = var.clamp(min=0.0)
        yt = y.transpose(1, 2)
        # (F.group_norm refuses one value per group; over a single frame it is F.layer_norm over time)
        want = (F.group_norm(yt, 512, None, None, R.CONV0_EPS) if frames > 1 else
                F.layer_norm(yt, (1,), None, None, R.CONV0_EPS)).transpose(1, 2)
        got = (y - mean[:, None]) / torch.sqrt(var[:, None] + R.CONV0_EPS)
        assert float((got - want).abs().max()) < 1e-7, frames


def test_conv0_reference_is_the_oracles_first_layer():
    """hubert_conv0 = conv0 -> GroupNorm -> GELU (HubertGroupNormConvLayer) and conv0 + bias -> LayerNorm -> GELU
    (HubertLayerNormConvLayer) in float64; with `frames`, GroupNorm over each clip's own first frames."""
    w0, gamma, beta, bias = R.conv0_weights(3)
    x = torch.stack([_normalised(R.speech_like(4005, s))[0] for s in (4, 5)])
    w = w0.double().view(512, 1, 10)
    y = F.conv1d(x.double()[:, None], w, stride=5)
    want = F.gelu(F.group_norm(y, 512, gamma.double(), beta.double(), 1e-5)).transpose(1, 2)
    got, _ = R.hubert_conv0(x, w0, gamma, beta)
    assert float((got - want).abs().max()) < 1e-12
    yb = F.conv1d(x.double()[:, None], w, bias.double(), stride=5).transpose(1, 2)
    want = F.gelu(F.layer_norm(yb, (512,), gamma.double(), beta.double(), 1e-5))
    got, _ = R.hubert_conv0(x, w0, gamma, beta, family="layer", bias=bias)
    assert float((got - want).abs().max()) < 1e-12
    got, _ = R.hubert_conv0(x, w0, gamma, beta, frames=[799, 300])
    for b, n in ((0, 799), (1, 300)):
        one = F.gelu(F.group_norm(y[b:b + 1, :, :n], 512, gamma.double(), beta.double(), 1e-5)).transpose(1, 2)[0]
        assert float((got[b, :n] - one).abs().max()) < 1e-12


def test_conv0_bound_rejects_the_statistics_mutations():
    """The GroupNorm-form bound is tight enough to tell apart, on a 5 s clip (15,999 frames): a variance divided by
    n - 1 (a relative change of 6e-5), and an eps of 1e-7 instead of 1e-5 (on the channels whose variance is near
    eps).  It holds the float64 reference itself and, for a DC offset 100x the noise (normalize off), the
    conditioning kappa = mean(A^2) / (var + eps) that the double moments must absorb stays within the bound's reach."""
    w0, gamma, beta, _ = R.conv0_weights(6)
    x = _normalised(R.speech_like(80000, 7))
    ref, bound = R.hubert_conv0(x, w0, gamma, beta)
    for kw in (dict(var_div=-1), dict(eps=1e-7)):
        mut, _ = R.hubert_conv0(x, w0, gamma, beta, **kw)
        assert float(((mut - ref).abs() / bound).max()) > 4, kw
    # the LayerNorm form's eps on quiet frames (amplitude 1e-3, no bias: the channel variance is ~1e-6 there)
    q = x * 1e-3
    ref, bound = R.hubert_conv0(q, w0, gamma, beta, family="layer")
    mut, _ = R.hubert_conv0(q, w0, gamma, beta, family="layer", eps=1e-6)
    assert float(((mut - ref).abs() / bound).max()) > 4
    # a DC offset 100x the noise: kappa is pinned, and the cancellation term it costs stays below 1e-5 of var + eps
    xd = R.speech_like(80000, 8, dc=100.0, noise=1.0)[None]
    y, A = R.conv0(xd, w0)
    kappa = float(((A ** 2).mean(1) / (y.var(1, unbiased=False) + R.CONV0_EPS)).max())
    assert 1e3 < kappa < 1e6, kappa
    assert (3 * 16000 + 100) * R.U53 * kappa < 1e-5


@pytest.mark.parametrize("family", ["base", "large", "large_gn", "data2vec"])
def test_hidden0_reference_is_the_oracle_at_layer_0(family):
    """hubert_hidden0 (the stage-by-stage restatement that carries the error bound) equals the oracle's hidden_states[0]
    in float64: hubert_hidden_states(layers=0) for the post-LN families, the input of layer 0 for the stable one."""
    from mertools_b200.synthetic import hubert_state_dict
    from oracle.encoders import hubert_hidden_states
    kw = dict(base={}, large=dict(large=True), large_gn=dict(large=True, group_norm=True),
              data2vec=dict(data2vec=True))[family]
    sd = R.fp16_exact_front_end(hubert_state_dict(seed=5, layers=1, **kw))
    sdt = {k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()}
    x = torch.stack([_normalised(R.speech_like(6407, s))[0] for s in (8, 9)])
    got, bound = R.hubert_hidden0(sd, x)
    heads = 16 if family.startswith("large") else 12
    want = hubert_hidden_states(sdt, x, layers=1 if family == "large" else 0, heads=heads, dtype=torch.float64)[0]
    assert got.shape == want.shape == (2, 19, 1024 if family.startswith("large") else 768)
    assert float((got - want).abs().max()) < 1e-10
    assert bool((bound > 0).all()) and float((bound / want.abs().clamp(min=1e-3)).median()) < 5e-2


# ---- transformer stack: one layer of mer_run_stack ----------------------------------------------------------------------
def _stack_case(family, tokens=None, scale=1.0):
    """(state dict, names, oracle hidden states in float64, cu, form kwargs) of a one- or two-layer synthetic model."""
    from mertools_b200 import synthetic as S
    from mertools_b200 import weights as W
    from oracle import encoders as E
    g = _g(40)
    if family == "vit":
        sd = S.vit_state_dict(seed=0, layers=1, scale=scale)
        n = tokens or 1
        hs = E.vit_hidden_states(sd, torch.rand(n, 3, 224, 224, generator=g) * 2 - 1, layers=1, dtype=torch.float64)
        return sd, W.VIT_NAMES, [h.reshape(-1, 768) for h in hs], [197 * i for i in range(n + 1)], dict(pre_ln=True)
    if family == "clip":
        sd = S.clip_vision_state_dict(seed=4, variant="b32", layers=1, scale=scale)
        n = tokens or 2
        sdt = {k: torch.as_tensor(v) for k, v in sd.items()}
        _, hs = E.clip_image_features(sdt, torch.rand(n, 3, 224, 224, generator=g) * 2 - 1, layers=1,
                                      dtype=torch.float64)
        return sd, W.CLIP_NAMES, [h.reshape(-1, 768) for h in hs], [50 * i for i in range(n + 1)], \
            dict(pre_ln=True, quick=True, eps=1e-5)
    if family in ("hubert", "hubert_stable"):
        stable = family == "hubert_stable"
        sd = S.hubert_state_dict(seed=1, layers=2, large=stable, scale=scale)
        sdt = {k: torch.as_tensor(v) for k, v in sd.items()}
        x = torch.stack([_normalised(R.speech_like(16000, s))[0] for s in (1, 2)])
        hs = E.hubert_hidden_states(sdt, x, layers=2, heads=16 if stable else 12, dtype=torch.float64)
        D = 1024 if stable else 768
        return sd, W.HUBERT_NAMES, [h.reshape(-1, D) for h in hs], [0, 49, 98], \
            dict(pre_ln=stable, eps=1e-5, heads=D // 64)
    lens = tokens or [1, 2, 64, 65]
    large = family == "roberta_large"
    sd = S.bert_state_dict(300, seed=2, layers=1, large=large, scale=scale, max_pos=514)
    sdt = {k: torch.as_tensor(v) for k, v in sd.items()}
    gen = np.random.default_rng(3)
    seqs = [np.concatenate([[0], gen.integers(1, 299, n - 2), [299]])[:n] if n > 1 else np.array([299]) for n in lens]
    eps, off = (1e-5, 2) if large else (1e-12, 0)
    hs = [torch.cat([h[0] for h in t]) for t in zip(*(E.bert_hidden_states(sdt, s, layers=1, heads=16 if large else 12, eps=eps,
                                                            position_offset=off, dtype=torch.float64) for s in seqs))]
    hs = [h.reshape(-1, 1024 if large else 768) for h in hs]
    return sd, W.BERT_NAMES, hs, [int(c) for c in np.cumsum([0] + list(lens))], \
        dict(pre_ln=False, eps=eps, heads=16 if large else 12)


@pytest.mark.parametrize("family", ["vit", "clip", "hubert", "hubert_stable", "bert", "roberta_large"])
def test_stack_layer_is_the_oracles_layer(family):
    """stack_layer without operand rounding is one layer of the oracle (vit_hidden_states, clip_image_features,
    hubert_hidden_states in both layer orders, bert_hidden_states) in float64, on the oracle's own input."""
    sd, names, hs, cu, kw = _stack_case(family)
    w = R.layer_from_state_dict(sd, names, 0)
    form = R.stack_form(None, max_seqlen=max(b - a for a, b in zip(cu, cu[1:])), **kw)
    got, bound = R.stack_layer(w, hs[0], cu, form)
    assert float((got - hs[1]).abs().max()) < 1e-12
    assert bool((bound > 0).all())


EMULATED = [("vit", "f16"), ("vit", "tf32"), ("clip", "f16"), ("hubert", "f16"), ("hubert", "bf16x3"),
            ("hubert_stable", "bf16x3"), ("bert", "f16"), ("bert", "bf16x3")]


@pytest.mark.parametrize("family,mode", EMULATED)
def test_stack_bound_covers_an_fp32_emulation(family, mode):
    """An fp32 evaluation of the layer that rounds every operand the stack stores (LN output, q | k | v, P, ctx, FC1
    output) to the form's format lands inside the bound of the float64 restatement."""
    sd, names, hs, cu, kw = _stack_case(family)
    w = {k: (R.operand(v.float(), R.STACK_OPERAND[mode]).double() if k.startswith("w_") else v)
         for k, v in R.layer_from_state_dict(sd, names, 0).items()}
    form = R.stack_form(mode, max_seqlen=max(b - a for a, b in zip(cu, cu[1:])), **kw)
    x = hs[0].float()
    ref, bound = R.stack_layer(w, x, cu, form)
    emu, _ = R.stack_layer(w, x, cu, form, emulate=True)
    ratio = float(((emu.double() - ref).abs() / bound).max())
    print(f"stack layer {family} {mode}: fp32 emulation at {ratio:.3f} of the bound")
    assert 1e-3 < ratio <= 1.0


def test_stack_bound_rejects_the_faults():
    """Each wiring fault of STACK_FAULTS, restated, leaves the bound by 4x or more on some element in a form the GPU test
    runs (two ViT frames in fp16; a BERT batch of 1, 2, 64 and 65 tokens in fp16 and split bf16; CLIP B/32 for the
    activation).  Not listed: erf <-> tanh GELU (<= 3e-4 apart, below fp16's own noise after FC2) and BERT <-> RoBERTa
    eps (1e-12 vs 1e-5 against unit variances): the GEMM epilogue and LayerNorm tests cover those."""
    cases = []
    for family, mode in (("vit", "f16"), ("bert", "f16"), ("bert", "bf16x3"), ("clip", "f16")):
        sd, names, hs, cu, kw = _stack_case(family, tokens=2 if family == "vit" else None)
        w = {k: (R.operand(v.float(), R.STACK_OPERAND[mode]).double() if k.startswith("w_") else v)
             for k, v in R.layer_from_state_dict(sd, names, 0).items()}
        form = R.stack_form(mode, max_seqlen=max(b - a for a, b in zip(cu, cu[1:])), **kw)
        x = hs[0].float()
        cases.append((f"{family} {mode}", w, x, cu, form) + R.stack_layer(w, x, cu, form))
    worst = {}
    for fault in R.STACK_FAULTS:
        for name, w, x, cu, form, ref, bound in cases:
            if fault == "stale_operand":
                if form["pre_ln"]:
                    continue
                tr = {}                       # LN1's copy of the layer before: its x after the attention half
                R.stack_layer(w, x, cu, form, trace=tr)
                got, _ = R.stack_layer(w, x, cu, form, op_in=tr["x1"])
            else:
                got, _ = R.stack_layer(w, x, cu, form, fault=fault)
            r = float(((got - ref).abs() / bound).max())
            if r > worst.get(fault, ("", 0.0))[1]:
                worst[fault] = (name, r)
    print("fault / bound: " + ", ".join(f"{k} {v[1]:.1f} ({v[0]})" for k, v in worst.items()))
    assert all(worst[f][1] >= 4 for f in R.STACK_FAULTS), worst


def test_stack_routes_follow_the_encoder_predicates():
    """stack_route at each boundary of encoder.cu / attention.cu / attention_f16.cu."""
    f16 = {1: "f16", 128: "f16", 129: "short", 208: "short", 209: "f16", 249: "f16", 250: "f16", 253: "f16", 254: "f16", 505: "f16", 506: "long", 4096: "long",
           4097: "fallback"}
    split = {1: "tc", 253: "tc", 254: "f16", 505: "f16", 506: "long", 4096: "long", 4097: "fallback"}
    for n, r in f16.items():
        assert R.stack_route("f16", n, long_rows=True) == r, n
    for n, r in split.items():
        assert R.stack_route("bf16x3", n, long_rows=True) == r, n
    assert R.stack_route("f16", 512) == "fallback" and R.stack_route("bf16x3", 512) == "fallback"   # BERT at 512
    assert R.stack_route("tf32", 197) == "tc" and R.stack_route("tf32", 257) == "f16"             # ViT / CLIP L/14


# ---- table-driven CNN executor ----------------------------------------------------------------------------------------
def test_cnn_operand_formats():
    x = torch.tensor([1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 65504.0, 65520.0, -1e30, 2.0 ** -25, float("nan")])
    got = R.f16_satfinite(x)
    assert got.tolist()[:7] == [1.0, 1.0, 1.0 + 2.0 ** -9, 65504.0, 65504.0, -65504.0, 0.0]      # ties to even, clamped
    assert math.isnan(got[7]) and got.dtype == torch.float32
    y = torch.randn(4096, generator=_g(20)) * 50
    hi, lo = R.split_bf16(y)
    assert torch.equal(hi, y.bfloat16().float()) and torch.equal(lo, (y - hi).bfloat16().float())
    assert bool(((y.double() - hi.double() - lo.double()).abs() <= 2.0 ** -16 * y.double().abs()).all())


def test_stem_operand_is_the_fused_multiply_add_then_the_division():
    """pix * scale - mean is exact in float64 for every 8-bit pixel (checked with fractions), so rounding it once to fp32
    is the fma; the plain fp32 product-then-subtract rounds twice and differs in some operands by an ulp."""
    from fractions import Fraction
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    scale = float(np.float32(1 / 255))
    for mv in mean:
        m32 = float(np.float32(mv))
        for pix in range(256):
            assert Fraction(pix * scale - m32) == Fraction(pix) * Fraction(scale) - Fraction(m32)
    frames = np.arange(256, dtype=np.uint8).repeat(3).reshape(1, 16, 16, 3)
    frames[..., 0] = frames[..., 0][:, ::-1]                    # different pixels in the three channels
    got = R.stem_operand(frames, 1 / 255, mean, std)
    rgb = torch.from_numpy(np.ascontiguousarray(frames[..., ::-1])).float()
    plain = (rgb * np.float32(1 / 255) - torch.tensor(mean)) / torch.tensor(std)
    # both round the difference once and the quotient once: they differ by at most an ulp of the operands' scale
    scale_ = (rgb.double() / 255 + torch.tensor(mean).double()) / torch.tensor(std).double()
    assert bool(((got - plain).double().abs() <= 2.0 ** -22 * scale_).all()) and int((got != plain).sum()) > 0
    exact = (rgb.double() / 255 - torch.tensor(mean).double()) / torch.tensor(std).double()
    assert float((got.double() - exact).abs().max()) < 1e-6


def test_cnn_conv_reference():
    x = torch.randn(2, 5, 4, 16, generator=_g(21)) * 3
    w = torch.randn(128, 3 * 3 * 16 + 8, generator=_g(22))      # padded columns past k k cin are ignored
    b = torch.randn(128, generator=_g(23))
    r = torch.randn(2, 3, 2, 128, generator=_g(24))
    y, a = R.cnn_conv(x, w, b, 3, 2, 1, res=r)
    wt = w[:, :144].reshape(128, 3, 3, 16).permute(0, 3, 1, 2).double()
    want = F.conv2d(x.permute(0, 3, 1, 2).double(), wt, b.double(), stride=2, padding=1).permute(0, 2, 3, 1) + r
    assert float((y - want).abs().max()) < 1e-12 and bool((a >= y.abs() - 1e-12).all())
    y16, _ = R.cnn_conv(x, w, b, 3, 2, 1, mode=R.GEMM_F16)
    want16, _ = R.cnn_conv(R.f16_satfinite(x), R.f16_satfinite(w), b, 3, 2, 1)
    assert torch.equal(y16, want16)
    ys, _ = R.cnn_conv(x, w, b, 3, 2, 1, mode=R.GEMM_BF16X3)
    (xh, xl), (wh, wl) = R.split_bf16(x), R.split_bf16(w)
    full, _ = R.cnn_conv(xh.double() + xl.double(), wh.double() + wl.double(), b, 3, 2, 1)
    lolo, _ = R.cnn_conv(xl, wl, torch.zeros(128), 3, 2, 1)
    assert float((ys - (full - lolo)).abs().max()) < 1e-9 and float((full - lolo - full).abs().max()) > 0


def test_cnn_plan_mirrors_the_executor_on_the_extractor_tables():
    """The workspace layout the GPU tests read buffers from equals mer_cnn_workspace_bytes on the FER+ / SENet, MA-Net and
    EmoNet tables at 1 and 3 frames."""
    import ctypes as C

    from mertools_b200 import _lib
    from mertools_b200 import encoders as En
    from mertools_b200 import synthetic as S
    dll = _lib.lib()
    dll.mer_cnn_workspace_bytes.restype = C.c_longlong
    dll.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    pack = lambda w, b: (1, 1)  # noqa: E731
    for m, _keep in (En.ferplus_resnet50_tables(S.ferplus_resnet50_state_dict(9), pack),
                     En.ferplus_resnet50_tables(S.ferplus_resnet50_state_dict(9, se=True), pack),
                     En.manet_tables(S.manet_state_dict(3), pack), En.emonet_tables(S.emonet_state_dict(3), pack)):
        for n in (1, 3):
            assert R.cnn_plan(m, n)[0]["total"] == dll.mer_cnn_workspace_bytes(C.byref(m), n)
