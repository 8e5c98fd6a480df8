"""Regression-only heads (output_dim1 = 0: the CMU-MOSI / MOSEI, SIMS / SIMSv2 and crossdim dataloaders) on the device.

Float64 parity of every utterance- and frame-level fusion kernel form at out1 = 0 under the per-element bounds of
test_fusion_kernels_gpu.py (fast / row kernels with both weight-gradient forms, the fused Adam step, the autograd
node's two halves, the frame-level net, with masks and grad clip); the null-operand rule (emos / emos_out may be NULL
at out1 = 0 and only then); out1 == out2 == 0 refused everywhere and the top-N net refusing out1 = 0; two data-parallel
ranks against one; and the CLI against the golden of the unmodified MERBench trainer on the other corpora."""
import os
import random
import socket
import types

import numpy as np
import pytest
import torch

import _kernel_refs as R
import test_fusion_kernels_gpu as K
from mertools_b200 import synthetic as S

pytestmark = pytest.mark.gpu

P, SEED = K.P, K.SEED
LR, WD = K.LR, K.WD


def _ref(sd, xs, p, km, val, upstream=None):
    """fusion_f64 at out1 = 0: the MSE loss and its gradient (as the upstream gradient 2 (vals - val) / B of vals_out,
    which is what d MSE / d param is), plus the gradients of ``upstream`` when given."""
    r = R.fusion_f64(sd, xs, p, km)
    vo = r["out"][2]
    B, H = vo.shape[0], r["out"][0].shape[1]
    d = vo - val.to(torch.float64)
    mse = float((d * d).sum() / B)
    zeros = (torch.zeros(B, H, dtype=torch.float64, device=vo.device), torch.zeros(B, 0, device=vo.device))
    res = dict(out=r["out"], loss=(0.0, mse, mse), grads=R.fusion_f64(sd, xs, p, km, upstream=(*zeros, 2 * d / B))["up"])
    if upstream is not None:
        res["up"] = R.fusion_f64(sd, xs, p, km, upstream=upstream)["up"]
    return res


def _close_grads(case, what, flat_views, ref, Kmax, depth):
    """K._close_grads without the two empty fc_out_1 tensors (nothing to compare; their shapes are checked)."""
    assert list(flat_views) == list(ref), "parameter order"
    assert flat_views["fc_out_1.weight"].numel() == 0 and flat_views["fc_out_1.bias"].numel() == 0
    live = {n: r for n, r in ref.items() if r.numel()}
    scale = max(float(g.abs().max()) for g in live.values())
    for n, r in live.items():
        K._close(case, f"{what} {n}", flat_views[n], r, scale, Kmax, depth)


def _check_losses(case, what, loss, ref, Kmax, depth):
    assert float(loss[0]) == 0.0, f"{case} {what}: the CE term of a regression-only head is 0"
    r = ref["loss"][1]
    K._close(case, f"{what} loss 1", loss[1:2], torch.tensor([r]), abs(r), Kmax, depth)
    assert float(loss[2]) == float(loss[1])


def _no_emo(B, device):
    return torch.zeros(B, dtype=torch.int64, device=device)   # never read at out1 = 0


UTT = [  # id, widths, hidden, out2, B, masks, clip, misaligned
    ("fast-B7", (768, 768, 768), 128, 1, 7, "hash", -1.0, False),
    ("fast-B129-ext-clip", (768, 768, 768), 128, 1, 129, "ext", 0.01, False),
    ("fast-out4", (96, 64, 128), 64, 4, 33, "hash", -1.0, False),
    ("general4-H256", (768, 768, 768), 256, 1, 32, "hash", -1.0, False),
    ("general8-H100-B200", (768, 768, 768), 100, 1, 200, "ext", -1.0, False),
    ("scalar-wgrad-6373-130-3", (6373, 130, 3), 64, 1, 32, "hash", 0.01, False),
    ("scalar-wgrad-misaligned-nodrop", (768, 768, 768), 128, 1, 7, "none", -1.0, True),
]


@pytest.mark.parametrize("widths,hidden,out2,B,masks,clip,misaligned", [pytest.param(*c[1:], id=c[0]) for c in UTT])
def test_utterance_forms_out1_0(cuda, request, widths, hidden, out2, B, masks, clip, misaligned):
    """forward_train, backward, mer_fusion_fwd_bwd + mer_fusion_adam and the fused mer_fusion_step at out1 = 0."""
    from mertools_b200.fusion import FusionNet
    case = "reg-only-" + request.node.callspec.id
    p = 0.0 if masks == "none" else P
    sd = S.fusion_state_dict(seed=3, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             out1=0, out2=out2)
    xs = K._inputs(widths, B, cuda, misaligned)
    _, val = K._labels(B, 1, out2, 5, cuda)
    emo = _no_emo(B, cuda)
    mw = list(widths) + [3 * hidden]
    km = None if masks == "none" else (K._hash_masks(SEED, 0, B, mw, cuda) if masks == "hash" else K._ext_masks(B, mw, cuda))
    ext = km if masks == "ext" else None
    ups = [K._randn((B, hidden), 200, cuda), torch.zeros(B, 0, device=cuda), K._randn((B, out2), 202, cuda)]
    ref = _ref(sd, xs, p, km, val, upstream=ups)
    Kmax = max(max(widths), 3 * hidden, B)

    def net():
        n = FusionNet(*widths, hidden, 0, out2, dropout=p, grad_clip=clip, device=cuda, max_batch=B, seed=SEED)
        return n.load_state_dict(sd)

    n = net()
    f, e, v = n.forward_train(*xs, ext_masks=ext)
    assert e.shape == (B, 0)
    K._close(case, "forward_train features", f, ref["out"][0], float(ref["out"][0].abs().max()), Kmax, K.DEPTH_MLP // 2)
    K._close(case, "forward_train vals", v, ref["out"][2], float(ref["out"][2].abs().max()), Kmax, K.DEPTH_MLP // 2)
    n.backward(*xs, *ups, ext_masks=ext)
    _close_grads(case, "backward", n.named_views(n.grads), ref["up"], Kmax, K.DEPTH_MLP)
    n.backward(*xs, ups[0], None, ups[2], ext_masks=ext)  # a NULL d_emos is the same thing
    _close_grads(case, "backward null d_emos", n.named_views(n.grads), ref["up"], Kmax, K.DEPTH_MLP)
    for fused in (False, True):
        n = net()
        p0 = n.params.clone()
        loss, eo, vo = n.train_step(*xs, emo, val, lr=LR, betas=K.BETAS, eps=K.EPS, weight_decay=WD, ext_masks=ext,
                                    use_graph=False, fused_adam=fused)
        what = "step" if fused else "fwd_bwd"
        assert eo.shape == (B, 0)
        _check_losses(case, what, loss, ref, Kmax, K.DEPTH_MLP // 2)
        K._close(case, f"{what} vals", vo, ref["out"][2], float(ref["out"][2].abs().max()), Kmax, K.DEPTH_MLP // 2)
        _close_grads(case, what, n.named_views(n.grads), ref["grads"], Kmax, K.DEPTH_MLP)
        assert int(n.step_counter) == 1
        K._adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, 1, clip=clip if clip != -1 else 0.0)
    n = net()
    loss_g, _, vo_g = n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, use_graph=True)
    if ext is None and not misaligned:   # the captured fused step gives the eager one's bits
        n2 = net()
        loss_e, _, vo_e = n2.train_step(*xs, emo, val, lr=LR, weight_decay=WD, use_graph=False)
        assert torch.equal(loss_g, loss_e) and torch.equal(vo_g, vo_e) and torch.equal(n.params, n2.params)
    K._report(case)


def test_autograd_node_out1_0(cuda):
    """get_models(args) for attention at output_dim1 = 0: MSE alone through the autograd node, against float64; the
    initial fc_out_1 is torch's nn.Linear(hidden, 0)."""
    from mertools_b200.fusion import get_models
    args = types.SimpleNamespace(model="attention", feat_type="utt", audio_dim=768, text_dim=768, video_dim=768,
                                 output_dim1=0, output_dim2=1, dropout=0.0, hidden_dim=64, grad_clip=-1.0, seed=0)
    torch.manual_seed(0)
    model = get_models(args).cuda()
    sd = {k: v.detach().cpu().clone() for k, v in model.model.state_dict().items()}
    torch.manual_seed(0)
    ref_sd = {}
    for e, d in (("audio_encoder", 768), ("text_encoder", 768), ("video_encoder", 768), ("attention_mlp", 192)):
        for l, k in (("linear_1", d), ("linear_2", 64), ("linear_3", 64)):
            ref_sd.update({f"{e}.{l}.{n}": v for n, v in torch.nn.Linear(k, 64).state_dict().items()})
    for l, o in (("fc_att", 3), ("fc_out_1", 0), ("fc_out_2", 1)):
        ref_sd.update({f"{l}.{n}": v for n, v in torch.nn.Linear(64, o).state_dict().items()})
    assert list(sd) == list(ref_sd) and all(torch.equal(sd[k], ref_sd[k]) for k in sd)
    assert sd["fc_out_1.weight"].shape == (0, 64)
    B = 9
    xs = [K._randn((B, 768), 800 + i, cuda) for i in range(3)]
    _, val = K._labels(B, 1, 1, 4, cuda)
    feats, eo, vo, _ = model({"audios": xs[0], "texts": xs[1], "videos": xs[2]})
    assert eo.shape == (B, 0)
    loss = torch.nn.functional.mse_loss(vo.view(-1, 1), val.view(-1, 1), reduction="sum") / B
    loss.backward()
    ref = _ref(sd, xs, 0.0, None, val)
    views = {n: p.grad for n, p in model.model.named_parameters()}
    _close_grads("reg-only-autograd", "grads", views, ref["grads"], 768, K.DEPTH_MLP)
    K._report("reg-only-autograd")


FRM = [("frm-H32-B1-hash", 32, (1, 2, 64), 1, "hash", -1.0), ("frm-H128-B300-ext-clip", 128, (2, 64, 1), 300, "ext", 0.01)]


@pytest.mark.parametrize("hidden,lens,B,masks,clip", [pytest.param(*c[1:], id=c[0]) for c in FRM])
def test_frame_level_out1_0(cuda, request, hidden, lens, B, masks, clip):
    from mertools_b200.fusion import FusionNet
    case = "reg-only-" + request.node.callspec.id
    widths = (64, 130, 3)
    sd = S.fusion_state_dict(seed=5, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             out1=0, out2=1, feat_type="frm_align")
    xs = [K._randn((B, T, w), 400 + i, cuda) for i, (T, w) in enumerate(zip(lens, widths))]
    _, val = K._labels(B, 1, 1, 7, cuda)
    mw = [hidden] * 3 + [3 * hidden]
    km = K._hash_masks(SEED, 0, B, mw, cuda) if masks == "hash" else K._ext_masks(B, mw, cuda)
    ref = _ref(sd, xs, P, km, val)
    n = FusionNet(*widths, hidden, 0, 1, dropout=P, grad_clip=clip, device=cuda, max_batch=B, seed=SEED,
                  feat_type="frm_align")
    n.load_state_dict(sd)
    p0 = n.params.clone()
    loss, eo, vo = n.train_step(*xs, _no_emo(B, cuda), val, lr=LR, weight_decay=WD,
                                ext_masks=km if masks == "ext" else None, use_graph=False)
    Kmax = max(max(widths), 4 * hidden, B * max(lens))
    depth = K.DEPTH_MLP + 2 * max(lens)
    assert eo.shape == (B, 0)
    _check_losses(case, "frm", loss, ref, Kmax, depth // 2)
    K._close(case, "vals", vo, ref["out"][2], float(ref["out"][2].abs().max()), Kmax, depth // 2)
    _close_grads(case, "fwd_bwd", n.named_views(n.grads), ref["grads"], Kmax, depth)
    K._adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, 1, clip=clip if clip != -1 else 0.0)
    f2, e2, v2, _ = n.train(False).forward({"audios": xs[0], "texts": xs[1], "videos": xs[2]})
    ref_v = R.fusion_f64(n.state_dict(), xs)["out"][2]
    assert e2.shape == (B, 0)
    K._close(case, "eval vals", v2, ref_v, float(ref_v.abs().max()), Kmax, depth // 2)
    K._report(case)


# ---- NULL emos / emos_out, and the refused head shapes ----------------------------------------------------------------
def _rcs(cuda, out1, out2, null_emos):
    """Return codes of every utterance / frame-level entry point and the top-N step at (out1, out2), with NULL emos /
    emos_out / d_emos when ``null_emos``."""
    import ctypes as C

    from mertools_b200 import _lib as L
    from mertools_b200.fusion import MerAdamHyper, MerFusionDims, MerFusionTopnDims
    B, H = 5, 64
    x = [K._randn((B, 96), 900 + i, cuda) for i in range(3)]
    emo, val = K._labels(B, 6, 1, 3, cuda)
    feats, emos, vals = (torch.empty(B, n, device=cuda) for n in (H, 6, 1))
    e_in, e_out = (None, None) if null_emos else (L.ptr(emo), L.ptr(emos))
    lib = L.lib()
    lib.mer_fusion_param_count.restype = lib.mer_fusion_frm_param_count.restype = C.c_longlong
    lib.mer_fusion_workspace_bytes.restype = lib.mer_fusion_frm_workspace_bytes.restype = C.c_longlong
    lib.mer_fusion_workspace_bytes.argtypes = [C.POINTER(MerFusionDims), C.c_int]
    lib.mer_fusion_frm_workspace_bytes.argtypes = [C.POINTER(MerFusionDims)] + [C.c_int] * 4
    dims = MerFusionDims(96, 96, 96, H, out1, out2)
    d = C.byref(dims)
    nbig = 4 * 96 * 96 * 12   # room for every parameter of either net at these widths
    params, grads, m, v = (torch.zeros(nbig, device=cuda) for _ in range(4))
    loss, step = torch.zeros(4, device=cuda), torch.zeros(1, dtype=torch.int32, device=cuda)
    ws = torch.empty(max(int(lib.mer_fusion_workspace_bytes(d, B)), 1 << 20), dtype=torch.uint8, device=cuda)
    st = L.stream_ptr()
    vp, i32, f32, i64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong
    fwd = L.declare("mer_fusion_forward", [C.POINTER(MerFusionDims), vp, vp, vp, vp, i32, vp, i64, vp, vp, vp, vp])
    fb = L.declare("mer_fusion_fwd_bwd", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, vp, vp, i32, f32, f32,
                                          C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp, vp])
    stp = L.declare("mer_fusion_step", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32,
                                        C.c_ulonglong, vp, vp, C.POINTER(MerAdamHyper), vp, i64, vp, vp, vp, vp, vp])
    fwf = L.declare("mer_fusion_frm_forward", [C.POINTER(MerFusionDims), vp, vp, vp, vp, i32, i32, i32, i32, vp, i64,
                                               vp, vp, vp, vp])
    fbf = L.declare("mer_fusion_frm_fwd_bwd", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, i32, i32, i32, vp, vp, i32,
                                               f32, f32, C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp, vp])
    xp = list(map(L.ptr, x))
    rcs = {}
    rcs["forward"] = fwd(d, L.ptr(params), *xp, B, L.ptr(ws), ws.numel(), L.ptr(feats), e_out, L.ptr(vals), st)
    rcs["fwd_bwd"] = fb(d, L.ptr(params), L.ptr(grads), *xp, e_in, L.ptr(val), B, 1.0 / B, 0.0, 0, L.ptr(step), None,
                        L.ptr(ws), ws.numel(), L.ptr(loss), L.ptr(feats), e_out, L.ptr(vals), st)
    hyper = MerAdamHyper(1e-3, 0.9, 0.999, 1e-8, 0.0, 0.0)
    rcs["step"] = stp(d, L.ptr(params), L.ptr(grads), L.ptr(m), L.ptr(v), *xp, e_in, L.ptr(val), B, 1.0 / B, 0.0, 0,
                      L.ptr(step), None, C.byref(hyper), L.ptr(ws), ws.numel(), L.ptr(loss), L.ptr(feats), e_out,
                      L.ptr(vals), st)
    wsf = torch.empty(max(int(lib.mer_fusion_frm_workspace_bytes(d, B, 1, 1, 1)), 1 << 20), dtype=torch.uint8,
                      device=cuda)
    rcs["frm_forward"] = fwf(d, L.ptr(params), *xp, 1, 1, 1, B, L.ptr(wsf), wsf.numel(), L.ptr(feats), e_out,
                             L.ptr(vals), st)
    rcs["frm_fwd_bwd"] = fbf(d, L.ptr(params), L.ptr(grads), *xp, 1, 1, 1, e_in, L.ptr(val), B, 1.0 / B, 0.0, 0,
                             L.ptr(step), None, L.ptr(wsf), wsf.numel(), L.ptr(loss), L.ptr(feats), e_out, L.ptr(vals),
                             st)
    tdims = MerFusionTopnDims(2, (C.c_int * 18)(96, 96), H, out1, out2)
    lib.mer_fusion_topn_workspace_bytes.restype = C.c_longlong
    lib.mer_fusion_topn_workspace_bytes.argtypes = [C.POINTER(MerFusionTopnDims), C.c_int]
    tstep = L.declare("mer_fusion_topn_step", [C.POINTER(MerFusionTopnDims), vp, vp, vp, vp, vp, i32, f32, f32,
                                               C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp, vp])
    wt = torch.empty(max(int(lib.mer_fusion_topn_workspace_bytes(C.byref(tdims), B)), 1 << 20), dtype=torch.uint8,
                     device=cuda)
    fp = (C.c_void_p * 2)(x[0].data_ptr(), x[1].data_ptr())
    rcs["topn"] = tstep(C.byref(tdims), L.ptr(params), L.ptr(grads), C.cast(fp, C.c_void_p), L.ptr(emo), L.ptr(val), B,
                        1.0 / B, 0.0, 0, L.ptr(step), None, L.ptr(wt), wt.numel(), L.ptr(loss), L.ptr(feats),
                        L.ptr(emos), L.ptr(vals), st)
    torch.cuda.synchronize()
    return rcs


@pytest.mark.parametrize("out1", [0, 6])
def test_null_emos_only_at_out1_0(cuda, out1):
    """mer_fusion_forward / _fwd_bwd / _step and the frame-level forward and fwd_bwd take NULL emos and emos_out when
    out1 == 0 and refuse them when out1 >= 1; the top-N step refuses out1 == 0 whatever its operands."""
    rcs = _rcs(cuda, out1, 1, null_emos=True)
    print(f"[reg-only] out1 {out1}, NULL emos: return codes {rcs}")
    topn = rcs.pop("topn")
    assert (topn == 0) == (out1 != 0), f"top-N: return code {topn} at out1 = {out1}"
    for name, rc in rcs.items():
        assert (rc == 0) == (out1 == 0), f"{name}: return code {rc} at out1 = {out1}"


def test_no_head_at_all_is_refused(cuda):
    """out1 == out2 == 0 is refused by every entry point, with or without emotion operands."""
    for null_emos in (False, True):
        rcs = _rcs(cuda, 0, 0, null_emos)
        print(f"[reg-only] out1 = out2 = 0: return codes {rcs}")
        assert all(rc != 0 for rc in rcs.values()), rcs


# ---- data parallelism at out1 = 0 ------------------------------------------------------------------------------------
DP_WIDTHS = (96, 128, 64)
DP_BATCHES = (27, 5)   # a 27-row batch splits 14 / 13 over two ranks; then a last batch of 5 (3 / 2)


def _dp_worker(rank, world, port, backend, out):
    import torch.distributed as dist

    from mertools_b200.fusion import FusionNet
    dev = torch.device("cuda", rank if torch.cuda.device_count() >= world else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    sd = S.fusion_state_dict(seed=8, audio_dim=DP_WIDTHS[0], text_dim=DP_WIDTHS[1], video_dim=DP_WIDTHS[2],
                             hidden=64, out1=0, out2=1)
    batches = []
    for i, n in enumerate(DP_BATCHES):
        xs = [K._randn((n, w), 1000 + 10 * i + j, dev) for j, w in enumerate(DP_WIDTHS)]
        _, val = K._labels(n, 1, 1, 20 + i, dev)
        batches.append((xs, _no_emo(n, dev), val))
    net = FusionNet(*DP_WIDTHS, 64, 0, 1, dropout=0.0, device=dev)
    if rank == 0:
        net.load_state_dict(sd)
    net.broadcast_from(0)
    losses = []
    for _ in range(2):
        for xs, emo, val in batches:
            mine = [x[rank::world].contiguous() for x in xs]
            loss, eo, _ = net.train_step(*mine, emo[rank::world].contiguous(), val[rank::world].contiguous(), lr=1e-3,
                                         weight_decay=1e-5, world_size=world, global_batch=len(emo))
            assert eo.shape[1] == 0
            losses.append(loss.clone())
    torch.cuda.synchronize()
    if rank == 0:
        ref = FusionNet(*DP_WIDTHS, 64, 0, 1, dropout=0.0, device=dev).load_state_dict(sd)
        ref_losses = []
        for _ in range(2):
            for xs, emo, val in batches:
                l, _, _ = ref.train_step(*xs, emo, val, lr=1e-3, weight_decay=1e-5, use_graph=False)
                ref_losses.append(l.clone())
        out["loss_diff"] = max(float((x - y).abs().max()) for x, y in zip(losses, ref_losses))
        out["loss0"] = float(ref_losses[0][2])
        out["ce"] = max(float(x[0]) for x in losses)
        out["param_rel"] = float((net.params - ref.params).norm() / ref.params.norm())
    dist.destroy_process_group()


def test_two_ranks_equal_one_rank_on_the_concatenated_batch_out1_0(cuda):
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_dp_worker, args=(2, port, backend, out), nprocs=2, join=True)
    out = dict(out)
    print(f"data-parallel regression-only fusion ({backend}): {out}")
    assert out["ce"] == 0.0
    assert out["loss_diff"] <= 1e-5 * max(1.0, out["loss0"]) and out["param_rel"] <= 1e-5


# ---- the CLI against the golden of the unmodified MERBench trainer -----------------------------------------------------
CORPORA = {"CMUMOSI": ((40, 12, 12), 1), "SIMS": ((40, 12, 12), 2), "IEMOCAPFour": ((50,), 3), "MELD": ((40, 12, 12), 4)}
UTT_ARGV = ["--feat_type=utt", "--audio_feature=synA-UTT", "--text_feature=synT-UTT", "--video_feature=synV-UTT"]
CLI = {
    "cmumosi_utt": ["--dataset=CMUMOSI", *UTT_ARGV],
    "sims_frm_align": ["--dataset=SIMS", "--feat_type=frm_align", "--audio_feature=synA-FRA",
                       "--text_feature=synT-FRA", "--video_feature=synV-FRA"],
    "iemocapfour_utt": ["--dataset=IEMOCAPFour", *UTT_ARGV],
    "meld_utt": ["--dataset=MELD", *UTT_ARGV],
    "crossdim_sims_cmumosi": ["--train_dataset=SIMS", "--test_dataset=CMUMOSI", *UTT_ARGV],
    "crossdis_iemocapfour_meld": ["--train_dataset=IEMOCAPFour", "--test_dataset=MELD", *UTT_ARGV],
}


@pytest.fixture(scope="module")
def corpora(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("merbench_gpu"))
    paths = {ds: S.write_merbench_corpus(os.path.join(root, ds), ds, n=n, seed=seed, frame_level=ds == "SIMS")
             for ds, (n, seed) in CORPORA.items()}
    return types.SimpleNamespace(PATH_TO_LABEL={d: p[0] for d, p in paths.items()},
                                 PATH_TO_FEATURES={d: p[1] for d, p in paths.items()})


@pytest.mark.parametrize("cfg_name", list(CLI))
def test_main_release_merbench_reproduces_the_unmodified_reference_run(cuda, tmp_path, corpora, cfg_name):
    """tests/golden/main_release_merbench_golden.npz holds ``runpy`` of the UNMODIFIED MERBench/main-release.py
    (make_golden_main_release_merbench.py: 3 epochs, dropout 0, batch 32, seeded with 0).  Same folds and sample
    order, same best epochs, losses within 1e-3 relative, the same result-file names."""
    from mertools_b200 import main_release as MR
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "main_release_merbench_golden.npz"))
    pre = f"{cfg_name}_"
    hyper = tmp_path / "hyper.yaml"
    hyper.write_text(str(g["hyper"]))
    args = MR.build_parser().parse_args(["--model=attention", *CLI[cfg_name], f"--hyper_path={hyper}",
                                         f"--epochs={int(g['epochs'])}", "--batch_size=32",
                                         f"--save_root={tmp_path}/saved", "--gpu=0"])
    torch.manual_seed(int(g["seed"]))
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    log = {}
    saved = MR.main(args, config=corpora, log=log)
    E, F = int(g["epochs"]), int(g[pre + "folds"])
    assert [args.output_dim1, args.output_dim2] == list(g[pre + "output_dims"])
    for f in range(F):
        assert log["eval_names"][f * E] == list(g[f"{pre}fold{f}_eval_names_epoch0"]), f"fold {f}: eval split / order"
        assert log["train_names"][f * E] == list(g[f"{pre}fold{f}_train_names_epoch0"]), f"fold {f}: train order"
    assert log["best_index"] == list(g[pre + "best_index"])
    rel = lambda a, b: np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max()  # noqa: E731
    tr, ev = np.array(log["train_loss"]).reshape(F, E), np.array(log["eval_loss"]).reshape(F, E)
    T = g[pre + "test_loss"].shape[0]
    msg = f"main-release MERBench golden {cfg_name}: train loss rel {rel(tr, g[pre + 'train_loss']):.2e}, " \
          f"eval {rel(ev, g[pre + 'eval_loss']):.2e}"
    assert rel(tr, g[pre + "train_loss"]) < 1e-3 and rel(ev, g[pre + "eval_loss"]) < 1e-3
    if T:
        ts = np.array(log["test_loss"]).reshape(F, E, T).transpose(2, 0, 1)
        msg += f", test {rel(ts, g[pre + 'test_loss']):.2e}"
        assert rel(ts, g[pre + "test_loss"]) < 1e-3
    print(msg)
    for f, best in enumerate(log["folder_save"]):
        for k in ("eval_emofscore", "eval_emoacc"):
            assert abs(best[k] - float(g[f"{pre}fold{f}_{k}"])) < 1e-9, (f, k)
    assert len(saved) == len(g[pre + "saved"])
    for path, ref in zip(saved, g[pre + "saved"]):
        assert os.path.basename(path).rsplit("_", 1)[0] == str(ref)
    assert ("-cross-" in saved[0]) == cfg_name.startswith("cross")
