"""CPU checks of tests/_kernel_refs.py: the float64 references the kernel-level GPU tests compare with are themselves
compared with torch's operators (or a second, independent formula) at small shapes."""
import numpy as np
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
