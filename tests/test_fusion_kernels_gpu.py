"""Kernel-level float64 parity of the fusion nets' training kernels: every form of the utterance-level row kernel and of
its weight-gradient kernel, the frame-level (LSTM) and top-N nets, the stand-alone Adam, and the counter-hash dropout
masks the benchmark and the trainer draw (tests/_kernel_refs.keep_mask restates the hash; fusion_f64 runs the oracle's
network in float64 on double copies of the kernels' fp32 operands).

Which form a case reaches follows launch_rows / launch_wgrad of csrc/fusion_fused.cu:
  fus_rows_fast_kernel   hidden <= 128 and a multiple of 32, out1 <= 8, every width a multiple of 4, plan <= 227 KB,
                         every input 16-byte aligned;
  fus_rows_kernel<8>     otherwise, when B >= 128 and hidden <= 128;  fus_rows_kernel<4> otherwise;
  fus_wgrad_kernel<1>    a width not a multiple of 4, or an operand row (input without dropout, features) not 16-byte
                         aligned;  fus_wgrad_kernel<4> otherwise.

Error bounds.  Every value the kernels produce is a chain of fp32 sums with round-to-nearest: dot products over the input
widths, the concat (3 H or N H) and H, and in a weight gradient a sum over the B (frame level: B T) rows.  A K-term sum
whose rounding errors are independent is off by about u sqrt(K) times the size of its terms (u = 2^-24; the
probabilistic bound of Higham & Mary, SIAM J. Sci. Comput. 41 (2019)); 4 of those is a per-sum bound that a fixed input
exceeds with negligible probability.  An error entering one layer leaves it with gain <= 1 at this initialisation
(uniform +-1/sqrt(fan_in) weights), so a value `depth` sums deep is off by at most depth times that:
    bound = 4 * depth * u * sqrt(K) * scale,
K the longest sum in the chain, depth the forward plus backward layer count (an LSTM adds its T steps each way), scale
the largest |float64 value| of the compared output, or for a gradient the largest |float64 gradient| of the whole net:
the backward carries absolute errors from the head down with gain <= 1, so a layer whose gradient is small (a bias sum
that cancels, an encoder the attention weights little) still holds the error of the layers above it."""
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import synthetic as S

pytestmark = pytest.mark.gpu

SEED, P = 11, 0.5
LR, BETAS, EPS, WD = 1e-3, (0.9, 0.999), 1e-8, 1e-5
DEPTH_MLP = 18          # 3 encoder + 3 attention-MLP layers, fc_att, the weighted sum and the heads; the same back
WORST = {}              # case -> (worst error / bound, where), printed at the end of each test


def _record(case, ratio, where):
    if ratio > WORST.get(case, (-1.0, ""))[0]:
        WORST[case] = (ratio, where)


def _bound(scale, K, depth):
    return 4 * depth * R.U32 * math.sqrt(K) * scale + 1e-30


def _close(case, what, got, ref, scale, K, depth):
    err = float((got.double() - ref.double().to(got.device)).abs().max())
    bound = _bound(scale, K, depth)
    _record(case, err / bound, what)
    assert err <= bound, f"{case} {what}: |err| {err:.3e} > bound {bound:.3e} (scale {scale:.3e})"


def _close_grads(case, what, flat_views, ref, K, depth):
    scale = max(float(g.abs().max()) for g in ref.values())   # see the module docstring
    assert list(flat_views) == list(ref), "parameter order"
    for n, r in ref.items():
        _close(case, f"{what} {n}", flat_views[n], r, scale, K, depth)


def _adam_close(case, p_new, p0, g, m_new, v_new, t, clip=0.0, grad_scale=1.0, m0=None, v0=None, lr=LR, wd=WD):
    """The Adam update against adam_f64 fed with the kernel's own gradient, elementwise, u = 2^-24 per rounding.  g' (the
    scaled, clipped gradient plus wd p) carries 2 roundings; m = fma(g' - m0, 1 - beta1, m0) adds 2 more, so m is off by
    <= 6 u (beta1 |m0| + (1 - beta1) |g'|); v = fma(v0, beta2, ((1 - beta2) g') g') doubles g''s 2 and adds 3: 8 u
    (beta2 v0 + (1 - beta2) g'^2).  The step lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps) adds 6 roundings of its own,
    sqrt(bc2) and bc1 one each, and powf(beta, t) (<= 4 ulp) enters through 1 - beta^t with relative errors
    4 u beta1^t / bc1 and 2 u beta2^t / bc2; v's error enters the step halved; p - step rounds once more (u |p|).
    12 u covers the step's own roundings."""
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    b1, b2, lr32 = f32(BETAS[0]), f32(BETAS[1]), f32(lr)
    z = torch.zeros_like(p0, dtype=torch.float64)
    m0 = z if m0 is None else m0.double()
    v0 = z if v0 is None else v0.double()
    pr, mr, vr = R.adam_f64(p0, g, m0, v0, t, lr, *BETAS, EPS, wd, grad_scale=grad_scale, clip=clip)
    gg = g.double() * f32(grad_scale)
    if clip > 0:
        gg = gg.clamp(-f32(clip), f32(clip))
    gg = (gg + f32(wd) * p0.double()).abs()
    mag_m = b1 * m0.abs() + (1 - b1) * gg
    mag_v = b2 * v0 + (1 - b2) * gg * gg
    u = R.U32
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    rel = 12 * u + 4 * u * b1 ** t / bc1 + 2 * u * b2 ** t / bc2
    denom = vr.sqrt() / math.sqrt(bc2) + f32(EPS)
    bound_m = 6 * u * mag_m + 1e-45
    bound_v = 8 * u * mag_v + 1e-45
    bound_p = u * pr.abs() + lr32 / bc1 * (mr.abs() * rel + bound_m + mr.abs() * bound_v / (2 * vr + 1e-300)) / denom
    for what, got, ref, bnd in (("m", m_new, mr, bound_m), ("v", v_new, vr, bound_v), ("param", p_new, pr, bound_p)):
        r = float(((got.double() - ref).abs() / bnd).max())
        _record(case, r, f"adam {what}")
        assert r <= 1.0, f"{case} adam {what}: worst error / bound {r:.3f}"


def _report(case):
    r, where = WORST[case]
    print(f"[fusion-f64] {case}: worst error / bound {r:.3f} ({where})")


def _randn(shape, seed, device):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(device)


def _hash_masks(seed, step, B, widths, device):
    """The keep-masks the kernels draw at this step counter, restated on the host (tensor m, element row * width + col)."""
    return [torch.from_numpy(R.keep_mask(seed, m, step, B * w, P).reshape(B, w).astype(np.float32)).to(device)
            for m, w in enumerate(widths)]


def _ext_masks(B, widths, device):
    g = torch.Generator().manual_seed(99)
    return [(torch.rand(B, w, generator=g) >= P).float().to(device) for w in widths]


def _labels(B, out1, out2, seed, device):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, out1, (B,), generator=g).to(device), (torch.rand(B, out2, generator=g) * 6 - 3).to(device)


# ---- utterance-level Attention ------------------------------------------------------------------------------------------
UTT = [  # id, (audio, text, video), hidden, out1, out2, B, masks, clip, misaligned inputs
    # fus_rows_fast_kernel + fus_wgrad_kernel<4>: 768 x 3, hidden 128, out1 6
    ("fast-B1", (768, 768, 768), 128, 6, 1, 1, "hash", -1.0, False),
    ("fast-B7", (768, 768, 768), 128, 6, 1, 7, "hash", -1.0, False),
    ("fast-B129-ext-clip", (768, 768, 768), 128, 6, 1, 129, "ext", 0.01, False),
    # fus_rows_kernel<4>: hidden 256 > 128
    ("general4-H256", (768, 768, 768), 256, 6, 1, 32, "hash", -1.0, False),
    # fus_rows_kernel<4>: the 3 x 8 x 4096 staging buffer leaves the 227 KB plan; B 32 < 128
    ("general4-wide-B32", (1024, 4096, 768), 128, 6, 1, 32, "hash", 0.01, False),
    # fus_rows_kernel<8>: same widths, B 300 >= 128 at hidden <= 128
    ("general8-wide-B300", (1024, 4096, 768), 128, 6, 1, 300, "hash", -1.0, False),
    # fus_rows_kernel<8>: hidden 100 is not a multiple of 32; B 200 >= 128
    ("general8-H100-B200", (768, 768, 768), 100, 6, 1, 200, "ext", -1.0, False),
    # fus_rows_kernel<4>: out1 16 > 8 (out2 4 rides along)
    ("general4-out16-out2-4", (768, 768, 768), 128, 16, 4, 32, "hash", -1.0, False),
    # fus_rows_kernel<4> + fus_wgrad_kernel<1>: widths not multiples of 4
    ("scalar-wgrad-6373-130-3", (6373, 130, 3), 64, 6, 1, 32, "hash", -1.0, False),
    # fus_rows_kernel<4> + fus_wgrad_kernel<1>: inputs one float off a 16-byte boundary (the fast kernel's 16-byte
    # staging loads would fault on them); no dropout, so W1's gradient reads the inputs themselves
    ("scalar-wgrad-misaligned", (768, 768, 768), 128, 6, 1, 7, "none", -1.0, True),
    # fus_rows_kernel<4>: hidden 4, the smallest accepted value
    ("general4-H4", (768, 768, 768), 4, 6, 1, 7, "hash", -1.0, False),
]
HASH_STEPS = {"fast-B7": (0, 41), "general4-wide-B32": (0, 41)}


def _utt_params():
    for c in UTT:
        for step in HASH_STEPS.get(c[0], (0,)):
            yield pytest.param(*c[1:], step, id=f"{c[0]}-step{step}")


def _inputs(widths, B, device, misaligned):
    xs = [_randn((B, w), 100 + i, device) for i, w in enumerate(widths)]
    if not misaligned:
        return xs
    out = []
    for x in xs:  # the same values one float past a 16-byte boundary
        buf = torch.empty(x.numel() + 1, device=device)
        v = buf[1:].view(x.shape)
        v.copy_(x)
        assert v.data_ptr() % 16 == 4
        out.append(v)
    return out


@pytest.mark.parametrize("widths,hidden,out1,out2,B,masks,clip,misaligned,step", list(_utt_params()))
def test_utterance_forms_against_float64(cuda, request, widths, hidden, out1, out2, B, masks, clip, misaligned, step):
    """forward_train, backward (upstream gradients), mer_fusion_fwd_bwd + mer_fusion_adam and the fused mer_fusion_step
    against float64 under the same masks: outputs, losses, all 28 gradient tensors and the Adam update."""
    from mertools_b200.fusion import FusionNet
    case = request.node.callspec.id
    p = 0.0 if masks == "none" else P
    sd = S.fusion_state_dict(seed=3, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             out1=out1, out2=out2)
    xs = _inputs(widths, B, cuda, misaligned)
    emo, val = _labels(B, out1, out2, 5, cuda)
    mw = list(widths) + [3 * hidden]
    km = None if masks == "none" else (_hash_masks(SEED, step, B, mw, cuda) if masks == "hash" else _ext_masks(B, mw, cuda))
    ext = km if masks == "ext" else None
    ups = [_randn((B, n), 200 + i, cuda) for i, n in enumerate((hidden, out1, out2))]
    ref = R.fusion_f64(sd, xs, p, km, emo, val, upstream=ups)
    K = max(max(widths), 3 * hidden, B)

    def net():
        n = FusionNet(*widths, hidden, out1, out2, dropout=p, grad_clip=clip, device=cuda, max_batch=B, seed=SEED)
        n.load_state_dict(sd)
        n.step_counter.fill_(step)
        return n

    # the autograd node's two halves
    n = net()
    out = n.forward_train(*xs, ext_masks=ext)
    for what, g, r in zip(("features", "emos", "vals"), out, ref["out"]):
        _close(case, f"forward_train {what}", g, r, float(r.abs().max()), K, DEPTH_MLP // 2)
    n.backward(*xs, *ups, ext_masks=ext)
    _close_grads(case, "backward", n.named_views(n.grads), ref["up"], K, DEPTH_MLP)

    # mer_fusion_fwd_bwd, then mer_fusion_adam (the data-parallel form) / the fused step
    for fused in (False, True):
        n = net()
        p0 = n.params.clone()
        loss, eo, vo = n.train_step(*xs, emo, val, lr=LR, betas=BETAS, eps=EPS, weight_decay=WD, ext_masks=ext,
                                    use_graph=False, fused_adam=fused)
        what = "step" if fused else "fwd_bwd"
        for i, nm in enumerate(("ce", "mse", "total")):
            r = ref["loss"][i]
            _close(case, f"{what} loss {nm}", loss[i:i + 1], torch.tensor([r]), abs(r), K, DEPTH_MLP // 2)
        _close(case, f"{what} emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), K, DEPTH_MLP // 2)
        _close(case, f"{what} vals", vo, ref["out"][2], float(ref["out"][2].abs().max()), K, DEPTH_MLP // 2)
        _close_grads(case, what, n.named_views(n.grads), ref["grads"], K, DEPTH_MLP)
        assert int(n.step_counter) == step + 1
        _adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, step + 1,
                    clip=clip if clip != -1 else 0.0)
    _report(case)


def test_hashed_step_counter_advanced_by_the_kernel(cuda):
    """Two fused steps: the second one's forward and backward both use the counter the first step's kernel advanced
    (step 1), on parameters the first step updated.  Checked for the fast and the general row kernel."""
    from mertools_b200.fusion import FusionNet
    for case, hidden in (("counter-fast", 128), ("counter-general4-H256", 256)):
        sd = S.fusion_state_dict(seed=3, hidden=hidden)
        B = 9
        xs = [_randn((B, 768), 300 + i, cuda) for i in range(3)]
        emo, val = _labels(B, 6, 1, 6, cuda)
        n = FusionNet(hidden_dim=hidden, dropout=P, device=cuda, max_batch=B, seed=SEED).load_state_dict(sd)
        n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, use_graph=False)
        assert int(n.step_counter) == 1
        sd1 = {k: v.detach().cpu().clone() for k, v in n.state_dict().items()}
        loss, eo, _ = n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, use_graph=False)
        ref = R.fusion_f64(sd1, xs, P, _hash_masks(SEED, 1, B, [768] * 3 + [3 * hidden], cuda), emo, val)
        K = max(768, 3 * hidden)
        _close(case, "emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), K, DEPTH_MLP // 2)
        _close_grads(case, "grads", n.named_views(n.grads), ref["grads"], K, DEPTH_MLP)
        # the masks of step 0 would not do: the comparison above tells the steps apart
        other = R.fusion_f64(sd1, xs, P, _hash_masks(SEED, 0, B, [768] * 3 + [3 * hidden], cuda), emo, val)
        assert float((eo.double() - other["out"][1]).abs().max()) > 100 * _bound(
            float(ref["out"][1].abs().max()), K, DEPTH_MLP // 2)
        _report(case)


def test_generic_and_scalar_forms_on_fast_eligible_dims(cuda):
    """MER_FUSION_GENERIC / MER_FUSION_WGRAD_SCALAR are read once per process: a fresh interpreter runs the fast-eligible
    B = 7 case through fus_rows_kernel<4> and fus_wgrad_kernel<1> against the same float64 bounds."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MER_FUSION_GENERIC="1", MER_FUSION_WGRAD_SCALAR="1")
    target = f"{os.path.abspath(__file__)}::test_utterance_forms_against_float64[fast-B7-step41]"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", target], cwd=root, env=env,
                       capture_output=True, text=True, timeout=600)
    print("\n".join(line for line in r.stdout.splitlines() if "[fusion-f64]" in line or "passed" in line))
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "1 passed" in r.stdout


# ---- frame-level Attention (LSTM encoders) ------------------------------------------------------------------------------
FRM = [  # id, hidden, (T_audio, T_text, T_video), B, masks
    ("frm-H32-B1", 32, (1, 2, 64), 1, "hash"),
    ("frm-H96-B300", 96, (64, 1, 2), 300, "hash"),
    ("frm-H128-B300-ext", 128, (2, 64, 1), 300, "ext"),
]


def _frm_params():
    for c in FRM:
        for step in ((0, 41) if c[4] == "hash" else (0,)):
            yield pytest.param(*c[1:], step, id=f"{c[0]}-step{step}")


@pytest.mark.parametrize("hidden,lens,B,masks,step", list(_frm_params()))
def test_frame_level_against_float64(cuda, request, hidden, lens, B, masks, step):
    """mer_fusion_frm_fwd_bwd + mer_fusion_adam: losses, outputs, all 24 gradient tensors and the update."""
    from mertools_b200.fusion import FusionNet
    case = request.node.callspec.id
    widths = (64, 130, 3)
    sd = S.fusion_state_dict(seed=5, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             feat_type="frm_align")
    xs = [_randn((B, T, w), 400 + i, cuda) for i, (T, w) in enumerate(zip(lens, widths))]
    emo, val = _labels(B, 6, 1, 7, cuda)
    mw = [hidden] * 3 + [3 * hidden]     # masks 0..2 act on the final hidden states
    km = _hash_masks(SEED, step, B, mw, cuda) if masks == "hash" else _ext_masks(B, mw, cuda)
    ref = R.fusion_f64(sd, xs, P, km, emo, val)
    n = FusionNet(*widths, hidden, 6, 1, dropout=P, device=cuda, max_batch=B, seed=SEED, feat_type="frm_align")
    n.load_state_dict(sd)
    n.step_counter.fill_(step)
    p0 = n.params.clone()
    loss, eo, vo = n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, ext_masks=km if masks == "ext" else None,
                                use_graph=False)
    K = max(max(widths), 4 * hidden, B * max(lens))
    depth = DEPTH_MLP + 2 * max(lens)
    _close(case, "loss total", loss[2:3], torch.tensor([ref["loss"][2]]), abs(ref["loss"][2]), K, depth // 2)
    _close(case, "emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), K, depth // 2)
    _close(case, "vals", vo, ref["out"][2], float(ref["out"][2].abs().max()), K, depth // 2)
    _close_grads(case, "fwd_bwd", n.named_views(n.grads), ref["grads"], K, depth)
    _adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, step + 1)
    _report(case)


# ---- Attention_TOPN -----------------------------------------------------------------------------------------------------
TOPN = [  # id, feature widths, hidden, B, masks
    ("topn-N1-H4", [6373], 4, 7, "hash"),
    ("topn-N2-H100", [1, 4096], 100, 33, "hash"),
    ("topn-N18-H256", [1, 3, 4096, 6373, 3, 1] * 3, 256, 20, "hash"),
    ("topn-N2-H100-ext", [3, 6373], 100, 33, "ext"),
]


def _topn_params():
    for c in TOPN:
        for step in ((0, 41) if c[4] == "hash" else (0,)):
            yield pytest.param(*c[1:], step, id=f"{c[0]}-step{step}")


@pytest.mark.parametrize("widths,hidden,B,masks,step", list(_topn_params()))
def test_topn_against_float64(cuda, request, widths, hidden, B, masks, step):
    """mer_fusion_topn_step + mer_fusion_adam: losses, outputs, every gradient tensor and the update."""
    from mertools_b200.fusion import TopnFusionNet
    case = request.node.callspec.id
    N = len(widths)
    sd = S.fusion_topn_state_dict(widths, seed=8, hidden=hidden)
    xs = [_randn((B, w), 500 + i, cuda) for i, w in enumerate(widths)]
    emo, val = _labels(B, 6, 1, 8, cuda)
    mw = list(widths) + [N * hidden]
    km = _hash_masks(SEED, step, B, mw, cuda) if masks == "hash" else _ext_masks(B, mw, cuda)
    ref = R.fusion_f64(sd, xs, P, km, emo, val)
    n = TopnFusionNet(widths, hidden, dropout=P, device=cuda, seed=SEED).load_state_dict(sd)
    n.step_counter.fill_(step)
    p0 = n.params.clone()
    loss, eo, vo = n.train_step(xs, emo, val, lr=LR, weight_decay=WD, ext_masks=km if masks == "ext" else None)
    K = max(max(widths), N * hidden, B)
    _close(case, "loss total", loss[2:3], torch.tensor([ref["loss"][2]]), abs(ref["loss"][2]), K, DEPTH_MLP // 2)
    _close(case, "emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), K, DEPTH_MLP // 2)
    _close(case, "vals", vo, ref["out"][2], float(ref["out"][2].abs().max()), K, DEPTH_MLP // 2)
    _close_grads(case, "topn_step", n.named_views(n.grads), ref["grads"], K, DEPTH_MLP)
    _adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, step + 1)
    _report(case)


# ---- mer_fusion_adam on its own -----------------------------------------------------------------------------------------
ADAM = [  # id, n, preset counter, grad_scale, clip, weight decay, zero moments / tiny gradients
    ("n1-t1", 1, 0, 1.0, 0.0, 0.0, False),
    ("n257-t1-scaled", 257, 0, 0.37, 0.0, 1e-5, False),
    ("n257-t10001-clip", 257, 10000, 1.0, 0.01, 0.0, False),
    ("n257-t10001-wd", 257, 10000, 2.0, 0.0, 1e-2, False),
    ("n257-eps-dominates", 257, 0, 1.0, 0.0, 0.0, True),
    ("n1-t10001-clip-wd-scaled", 1, 10000, 0.5, 0.02, 1e-3, False),
]


@pytest.mark.parametrize("n,counter,scale,clip,wd,tiny", [pytest.param(*c[1:], id=c[0]) for c in ADAM])
def test_adam_against_float64(cuda, request, n, counter, scale, clip, wd, tiny):
    from mertools_b200 import _lib as L
    from mertools_b200.fusion import TopnFusionNet
    case = "adam-" + request.node.callspec.id
    adam = TopnFusionNet([4], 4, device=cuda)._adam
    p = _randn((n,), 600, cuda)
    g = _randn((n,), 601, cuda) * (1e-12 if tiny else 0.05)
    if tiny:  # zero moments and a gradient whose sqrt(v) is far below eps
        m, v = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    else:
        m = _randn((n,), 602, cuda) * 0.01
        v = _randn((n,), 603, cuda).abs() * 1e-4
    counter_t = torch.full((1,), counter, dtype=torch.int32, device=cuda)
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    L.check(adam(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), n, LR, *BETAS, EPS, wd, scale, clip, L.ptr(counter_t),
                 L.stream_ptr()))
    assert int(counter_t) == counter + 1
    _adam_close(case, p, p0, g, m, v, counter + 1, clip=clip, grad_scale=scale, m0=m0, v0=v0, wd=wd)
    _report(case)


# ---- data parallelism with hashed dropout -------------------------------------------------------------------------------
DP_B = 13


def _dp_worker(rank, world, port, backend, mode, out):
    import torch.distributed as dist

    from mertools_b200.fusion import FusionNet
    dev = torch.device("cuda", rank if torch.cuda.device_count() >= world else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    sd = S.fusion_state_dict(seed=3, hidden=64)
    xs = [_randn((DP_B, 768), 700 + i, dev) for i in range(3)]       # the same rows on every rank
    emo, val = _labels(DP_B, 6, 1, 9, dev)
    net = FusionNet(hidden_dim=64, dropout=P, device=dev, max_batch=DP_B, seed=SEED)
    net.load_state_dict(sd)
    net.broadcast_from(0)
    _, eo, _ = net.train_step(*xs, emo, val, lr=LR, weight_decay=WD, world_size=world, global_batch=world * DP_B)
    eo_all = [torch.empty_like(eo) for _ in range(world)]
    dist.all_gather(eo_all, eo.contiguous())
    if rank == 0 and mode == "masks":
        out["emos_diff"] = float((eo_all[0] - eo_all[1]).abs().max())
    if rank == 0 and mode == "grads":
        from mertools_b200.fusion import rank_dropout_seed
        mw = [768] * 3 + [3 * 64]
        per_rank = [_hash_masks(rank_dropout_seed(SEED, r, world), 0, DP_B, mw, dev) for r in range(world)]
        masks = [torch.cat([pr[m] for pr in per_rank]) for m in range(4)]
        cat = lambda t: torch.cat([t] * world)  # noqa: E731
        ref = R.fusion_f64(sd, [cat(x) for x in xs], P, masks, cat(emo), cat(val))
        case = "dp-allreduced-grads"
        _close_grads(case, "all-reduced", net.named_views(net.grads), ref["grads"], 768, DEPTH_MLP)
        for r in range(world):
            _close(case, f"rank {r} emos", eo_all[r], ref["out"][1][r * DP_B:(r + 1) * DP_B],
                   float(ref["out"][1].abs().max()), 768, DEPTH_MLP // 2)
        out["worst"] = WORST[case]
    dist.destroy_process_group()


def _spawn_dp(mode):
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_dp_worker, args=(2, port, backend, mode, out), nprocs=2, join=True)
    return dict(out)


def test_data_parallel_ranks_draw_different_masks(cuda):
    """Two ranks holding the same rows and the same parameters: with dropout their train-mode outputs must differ.  With
    one shared seed the masks hash only (seed, tensor, step, local index), and every rank dropped the same elements."""
    out = _spawn_dp("masks")
    print(f"[fusion-dp] max |emos rank 0 - emos rank 1| = {out['emos_diff']:.3e}")
    assert out["emos_diff"] > 1e-2, "the data-parallel ranks drew identical dropout masks"


def test_data_parallel_allreduced_gradient_is_the_concatenated_batch_gradient(cuda):
    """The all-reduced gradient is the float64 gradient of the concatenated batch (rank 0's rows, then rank 1's) under
    each rank's restated masks, drawn from rank_dropout_seed(seed, rank, 2)."""
    out = _spawn_dp("grads")
    r, where = out["worst"]
    print(f"[fusion-f64] dp-allreduced-grads: worst error / bound {r:.3f} ({where})")
    assert r <= 1.0
