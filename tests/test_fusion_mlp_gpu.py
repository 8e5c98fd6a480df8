"""GPU tests of the MER2023 baseline nets (csrc/fusion_mlp.cu through mertools_b200.fusion_mlp.MlpFusionNet):
float64 parity with per-element bounds for the forward pass, the losses, every parameter's gradient and the Adam step
over both kinds, depths 1 / 2 / 3 / 8, widths 1 / 3 / 130 / 1024, input widths that are not multiples of 4, batches
1 (MLP) / 2 / 5 / 32 / 33, and hashed and injected keep-masks; bit-identical repeats (eager and CUDA graph); the golden of
MER2023/main-release.py replayed through the CLI; the refusal messages of the C ABI.

Error bounds as in test_fusion_kernels_gpu.py: a K-term fp32 sum is off by about u sqrt(K) times its terms, 4 of those
bound a sum, and an error crosses a layer with gain <= 1 at torch's initialisation, so
    bound = 4 * depth * u * sqrt(K) * scale,
K the longest sum of the net (the widest input, layer or the batch for a weight gradient), depth the forward plus
backward layer count (2 per layer of every chain on the path, plus the head), scale the largest |float64 value| of the
compared output, or for a gradient the largest |float64 gradient| of the whole net."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import _kernel_refs as R
import _mer2023_replay as RP
from mertools_b200 import _lib as L
from mertools_b200.fusion_mlp import MerMlpDims, MlpFusionNet, mask_shapes, reference_init
from oracle import mer2023 as O

pytestmark = pytest.mark.gpu
P, SEED, LR, WD = 0.3, 1234, 1e-3, 1e-5

# (kind, layers, input widths, batch, masks): every depth, width and batch the issue lists at least once per kind
CASES = [
    ("mlp", [256, 128], (10, 12, 7), 32, "hash"),
    ("mlp", [1], (3, 5, 1), 1, "ext"),
    ("mlp", [3, 130], (1582, 88, 17), 33, "hash"),
    ("mlp", [130, 1024, 3], (5, 6, 7), 5, "ext"),
    ("mlp", [64, 48, 40, 32, 24, 16, 8, 4], (9, 11, 13), 2, "hash"),
    ("mlp", [1024], (2048, 1024, 771), 33, "ext"),
    ("attention", [24, 16, 8], (10, 12, 7), 32, "hash"),
    ("attention", [1], (3, 5, 1), 2, "ext"),
    ("attention", [130, 3], (1582, 88, 17), 33, "hash"),
    ("attention", [1024, 130], (5, 6, 7), 5, "ext"),
    ("attention", [16, 16, 12, 12, 8, 8, 4, 3], (9, 11, 13), 32, "ext"),
    ("attention", [1024], (1025, 300, 771), 5, "hash"),
]


def _cid(c):
    return f"{c[0]}-{'x'.join(map(str, c[1]))}-in{'_'.join(map(str, c[2]))}-b{c[3]}-{c[4]}"


def _setup(case, seed=SEED):
    kind, layers, dims, B, mode = case
    torch.manual_seed(seed)
    sd = reference_init(kind, *dims, layers)
    g = torch.Generator().manual_seed(seed + 1)
    x = [torch.randn(B, d, generator=g) for d in dims]
    emo = torch.randint(0, 6, (B,), generator=g)
    val = torch.empty(B, 1).uniform_(-3, 3, generator=g)
    shapes = mask_shapes(kind, layers, B)
    if mode == "ext":
        masks = [torch.rand(s, generator=g) >= P for s in shapes]
    else:   # the counter hash at step 0, element row * width + col of mask t
        masks = [torch.from_numpy(R.keep_mask(SEED, t, 0, s[0] * s[1], P).reshape(s)) for t, s in enumerate(shapes)]
    return sd, x, emo, val, masks


def _f64(kind, sd, x, emo, val, masks):
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    feats, eo, vo = O.forward(sd64, kind, *[t.double() for t in x], masks=[m.double() for m in masks], p=P)
    ce, mse = O.losses(eo, vo, emo, val.double())
    grads = torch.autograd.grad(ce + mse, list(sd64.values()))
    return (feats.detach(), eo.detach(), vo.detach()), (float(ce), float(mse), float(ce + mse)), \
        dict(zip(sd64, grads))


def _bound(scale, K, depth):
    return 4 * depth * R.U32 * math.sqrt(K) * scale + 1e-30


def _net(kind, layers, dims, sd, seed=SEED):
    return MlpFusionNet(kind, *dims, layers, dropout=P, device="cuda", max_batch=64, seed=seed).load_state_dict(sd)


@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_step_vs_float64(case):
    kind, layers, dims, B, mode = case
    sd, x, emo, val, masks = _setup(case)
    net = _net(kind, layers, dims, sd)
    dev = [t.cuda() for t in x]
    ext = [m.float().cuda() for m in masks] if mode == "ext" else None
    loss, feats, eo, vo = net.train_step(*dev, emo.cuda(), val.cuda(), lr=LR, weight_decay=WD, ext_masks=ext,
                                         update=False)
    torch.cuda.synchronize()
    (rf, re, rv), rl, rg = _f64(kind, sd, x, emo, val, masks)
    K = max(max(dims) * (3 if kind == "mlp" else 1), 3 * layers[-1], max(layers), B)
    depth = 2 * len(layers) * (2 if kind == "attention" else 1) + 6
    for what, got, ref in (("features", feats, rf), ("emos", eo, re), ("vals", vo, rv)):
        err = float((got.cpu().double() - ref).abs().max())
        bound = _bound(float(ref.abs().max()), K, depth)
        assert err <= bound, f"{_cid(case)} {what}: {err:.3e} > {bound:.3e}"
    lg = loss.cpu().double()
    for i, what in enumerate(("ce", "mse", "total")):
        assert abs(float(lg[i]) - rl[i]) <= _bound(max(abs(rl[i]), 1.0), K, depth), f"{_cid(case)} loss {what}"
    scale = max(float(g.abs().max()) for g in rg.values())
    views = net.named_views(net.grads)
    assert list(views) == list(rg)
    for n, r in rg.items():
        err = float((views[n].cpu().double() - r).abs().max())
        bound = _bound(scale, K, depth)
        assert err <= bound, f"{_cid(case)} grad {n}: {err:.3e} > {bound:.3e} (scale {scale:.3e})"
    # the Adam step, fed with the kernel's own gradient (mer_fusion_adam's own bound is in test_fusion_kernels_gpu.py)
    p0, g0 = net.params.clone(), net.grads.clone()
    net.train_step(*dev, emo.cuda(), val.cuda(), lr=LR, weight_decay=WD, ext_masks=ext)
    torch.cuda.synchronize()
    assert torch.equal(net.grads, g0), "the update step recomputed a different gradient"
    z = torch.zeros_like(p0)
    p_ref, _, _ = R.adam_f64(p0.cpu(), g0.cpu(), z.cpu(), z.cpu(), 1, LR, 0.9, 0.999, 1e-8, WD)
    err = (net.params.cpu().double() - p_ref).abs()
    assert float((err - (24 * R.U32 * (p_ref.abs() + LR))).max()) <= 0, f"{_cid(case)} Adam step"
    assert int(net.step_counter.item()) == 1


@pytest.mark.parametrize("case", [CASES[0], CASES[6]], ids=_cid)
def test_repeat_runs_are_bit_identical(case):
    """Three steps with hashed masks, twice from the same state, eager and through the CUDA graph: same bits."""
    kind, layers, dims, B, _ = case
    sd, x, emo, val, _ = _setup(case)
    dev = [t.cuda() for t in x] + [emo.cuda(), val.cuda()]
    outs = []
    for use_graph in (False, True, True):
        net = _net(kind, layers, dims, sd)
        for _ in range(3):
            loss, f, eo, vo = net.train_step(*dev, lr=LR, weight_decay=WD, use_graph=use_graph)
        ev = net(*dev[:3])
        outs.append([t.clone() for t in (loss, f, eo, vo, net.params, net.exp_avg, net.exp_avg_sq, *ev)])
    torch.cuda.synchronize()
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


@pytest.mark.parametrize("tag", ["mlp", "att"])
def test_golden_replayed_through_the_cli(tag, tmp_path):
    """The CLI's host loop on MlpFusionNet with the reference's initial weights, sample orders and keep-masks."""
    def make(kind, dims, sd):
        return MlpFusionNet(kind, *dims, layers, dropout=P, device="cuda", max_batch=32).load_state_dict(sd)
    layers = "256,128" if tag == "mlp" else "24,16,8"
    rp, written, folder_save, name_time, args = RP.run(tag, str(tmp_path), make_net=make,
                                                       device=torch.device("cuda", 0), mask_device="cuda",
                                                       mask_dtype=torch.float32)
    assert args.layers == layers
    RP.check_replay(tag, rp, written, folder_save, name_time, args, str(tmp_path), tol=1e-4)


def _dims(kind=0, layers=(8, 4), ins=(5, 6, 7), out1=6, out2=1):
    lay = (C.c_int * 8)(*(list(layers[:8]) + [0] * (8 - len(layers[:8]))))
    return MerMlpDims(kind, *ins, len(layers), lay, out1, out2)


@pytest.mark.parametrize("dims, msg", [
    (_dims(kind=2), "kind 2 is neither"),
    (_dims(layers=()), "0 layers (1..8)"),
    (_dims(layers=(4,) * 9), "9 layers (1..8)"),
    (_dims(layers=(8, 0)), "layer 1 has width 0 (1..1024)"),
    (_dims(layers=(1025,)), "layer 0 has width 1025 (1..1024)"),
    (_dims(ins=(5, 0, 7)), "input width 0 of modality 1"),
    (_dims(ins=(65537, 6, 7)), "input width 65537 of modality 0"),
    (_dims(out1=0), "out1 0 (1..16"),
    (_dims(out1=17), "out1 17 (1..16"),
    (_dims(out2=0), "out2 0 (1..4"),
    (_dims(out2=5), "out2 5 (1..4"),
])
def test_refusals(dims, msg):
    lib = L.lib()
    lib.mer_mlp_param_count.restype = C.c_longlong
    lib.mer_mlp_param_count.argtypes = [C.POINTER(MerMlpDims)]
    assert lib.mer_mlp_param_count(C.byref(dims)) == -1
    assert msg in lib.mer_last_error().decode()


def test_refusals_of_batches_and_operands():
    lib = L.lib()
    lib.mer_mlp_workspace_bytes.restype = C.c_longlong
    lib.mer_mlp_workspace_bytes.argtypes = [C.POINTER(MerMlpDims), C.c_int]
    assert lib.mer_mlp_workspace_bytes(C.byref(_dims(kind=1)), 1) == -1
    assert "the Attention net needs at least 2 rows" in lib.mer_last_error().decode()
    assert lib.mer_mlp_workspace_bytes(C.byref(_dims(kind=0)), 0) == -1
    assert "batch 0 out of range" in lib.mer_last_error().decode()
    assert lib.mer_mlp_workspace_bytes(C.byref(_dims(kind=0)), 1) > 0
    net = _net("mlp", [8, 4], (5, 6, 7), reference_init("mlp", 5, 6, 7, [8, 4]))
    x = [torch.zeros(2, d, device="cuda") for d in (5, 6, 7)]
    fwd = L.declare("mer_mlp_forward", [C.POINTER(MerMlpDims)] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p,
                                                                                     C.c_longlong] + [C.c_void_p] * 4)
    rc = fwd(C.byref(net.dims), L.ptr(net.params), L.ptr(x[0]), L.ptr(x[1]), L.ptr(x[2]), 2, L.ptr(net.ws), 16,
             L.ptr(x[0]), L.ptr(x[0]), L.ptr(x[0]), L.stream_ptr())
    assert rc != 0 and "workspace of 16 bytes" in lib.mer_last_error().decode()
    rc = fwd(C.byref(net.dims), L.ptr(net.params), None, L.ptr(x[1]), L.ptr(x[2]), 2, L.ptr(net.ws),
             net.ws.numel(), L.ptr(x[0]), L.ptr(x[0]), L.ptr(x[0]), L.stream_ptr())
    assert rc != 0 and "null operand" in lib.mer_last_error().decode()
    att = _net("attention", [4], (5, 6, 7), reference_init("attention", 5, 6, 7, [4]))
    with pytest.raises(ValueError, match="at least 2 rows"):
        att(*[t[:1] for t in x])
