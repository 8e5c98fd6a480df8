"""Emotion-only heads (output_dim2 = 0: the MER2024 / MER2025 / MER2026 dataloaders) on the device.

Float64 parity of every fusion kernel form at out2 = 0 under the per-element bounds of test_fusion_kernels_gpu.py
(utterance fast / row kernels with both weight-gradient forms, the autograd node's two halves, the frame-level and the
top-N nets, each with the parameters after Adam); the null-operand rule (vals / vals_out may be NULL at out2 = 0 and
only then); the CLI against the golden of the unmodified MER2026 trainer; and top-N under data parallelism."""
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


def _close_grads(case, what, flat_views, ref, Kmax, depth):
    """K._close_grads without the two empty fc_out_2 tensors (nothing to compare; their shapes are checked)."""
    assert list(flat_views) == list(ref), "parameter order"
    assert flat_views["fc_out_2.weight"].numel() == 0 and flat_views["fc_out_2.bias"].numel() == 0
    live = {n: r for n, r in ref.items() if r.numel()}
    scale = max(float(g.abs().max()) for g in live.values())
    for n, r in live.items():
        K._close(case, f"{what} {n}", flat_views[n], r, scale, Kmax, depth)


def _empty_vals(B, device):
    return torch.zeros(B, 0, device=device)


def _check_losses(case, what, loss, ref, Kmax):
    assert float(loss[1]) == 0.0, f"{case} {what}: the MSE term of an emotion-only head is 0"
    for i in (0, 2):
        r = ref["loss"][i]
        K._close(case, f"{what} loss {i}", loss[i:i + 1], torch.tensor([r]), abs(r), Kmax, K.DEPTH_MLP // 2)
    assert float(loss[2]) == float(loss[0])


UTT = [  # id, widths, hidden, out1, B, masks, clip, misaligned
    ("fast-B7", (768, 768, 768), 128, 6, 7, "hash", -1.0, False),
    ("fast-B129-ext-clip", (768, 768, 768), 128, 6, 129, "ext", 0.01, False),
    ("general4-H256", (768, 768, 768), 256, 6, 32, "hash", -1.0, False),
    ("general8-H100-B200", (768, 768, 768), 100, 6, 200, "ext", -1.0, False),
    ("general4-out16", (768, 768, 768), 128, 16, 32, "hash", 0.01, False),
    ("scalar-wgrad-6373-130-3", (6373, 130, 3), 64, 6, 32, "hash", -1.0, False),
    ("scalar-wgrad-misaligned-nodrop", (768, 768, 768), 128, 6, 7, "none", -1.0, True),
]


@pytest.mark.parametrize("widths,hidden,out1,B,masks,clip,misaligned", [pytest.param(*c[1:], id=c[0]) for c in UTT])
def test_utterance_forms_out2_0(cuda, request, widths, hidden, out1, B, masks, clip, misaligned):
    """forward_train, backward, mer_fusion_fwd_bwd + mer_fusion_adam and the fused mer_fusion_step at out2 = 0."""
    from mertools_b200.fusion import FusionNet
    case = "emo-only-" + request.node.callspec.id
    p = 0.0 if masks == "none" else P
    sd = S.fusion_state_dict(seed=3, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             out1=out1, out2=0)
    xs = K._inputs(widths, B, cuda, misaligned)
    emo, _ = K._labels(B, out1, 0, 5, cuda)
    val = _empty_vals(B, cuda)
    mw = list(widths) + [3 * hidden]
    km = None if masks == "none" else (K._hash_masks(SEED, 0, B, mw, cuda) if masks == "hash" else K._ext_masks(B, mw, cuda))
    ext = km if masks == "ext" else None
    ups = [K._randn((B, n), 200 + i, cuda) for i, n in enumerate((hidden, out1))] + [_empty_vals(B, cuda)]
    ref = R.fusion_f64(sd, xs, p, km, emo, val, upstream=ups)
    Kmax = max(max(widths), 3 * hidden, B)

    def net():
        n = FusionNet(*widths, hidden, out1, 0, dropout=p, grad_clip=clip, device=cuda, max_batch=B, seed=SEED)
        return n.load_state_dict(sd)

    n = net()
    f, e, v = n.forward_train(*xs, ext_masks=ext)
    assert v.shape == (B, 0)
    K._close(case, "forward_train features", f, ref["out"][0], float(ref["out"][0].abs().max()), Kmax, K.DEPTH_MLP // 2)
    K._close(case, "forward_train emos", e, ref["out"][1], float(ref["out"][1].abs().max()), Kmax, K.DEPTH_MLP // 2)
    n.backward(*xs, *ups, ext_masks=ext)
    _close_grads(case, "backward", n.named_views(n.grads), ref["up"], Kmax, K.DEPTH_MLP)
    n.backward(*xs, ups[0], ups[1], None, ext_masks=ext)  # a NULL d_vals is the same thing
    _close_grads(case, "backward null d_vals", n.named_views(n.grads), ref["up"], Kmax, K.DEPTH_MLP)
    for fused in (False, True):
        n = net()
        p0 = n.params.clone()
        loss, eo, vo = n.train_step(*xs, emo, val, lr=LR, betas=K.BETAS, eps=K.EPS, weight_decay=WD, ext_masks=ext,
                                    use_graph=False, fused_adam=fused)
        what = "step" if fused else "fwd_bwd"
        assert vo.shape == (B, 0)
        _check_losses(case, what, loss, ref, Kmax)
        K._close(case, f"{what} emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), Kmax, K.DEPTH_MLP // 2)
        _close_grads(case, what, n.named_views(n.grads), ref["grads"], Kmax, K.DEPTH_MLP)
        assert int(n.step_counter) == 1
        K._adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, 1, clip=clip if clip != -1 else 0.0)
    # the graph-captured fused step (the trainer's path) gives the same bits as the eager one; its static input buffers
    # are 16-byte aligned, so misaligned inputs reach other kernel forms there and are left out
    n = net()
    loss_g, eo_g, _ = n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, ext_masks=None, use_graph=True)
    if ext is None and not misaligned:
        n2 = net()
        loss_e, eo_e, _ = n2.train_step(*xs, emo, val, lr=LR, weight_decay=WD, use_graph=False)
        assert torch.equal(loss_g, loss_e) and torch.equal(eo_g, eo_e) and torch.equal(n.params, n2.params)
    K._report(case)


def test_autograd_node_out2_0(cuda):
    """get_models(args) for attention at output_dim2 = 0: CE alone through the autograd node, against float64."""
    from mertools_b200.fusion import get_models
    args = types.SimpleNamespace(model="attention", feat_type="utt", audio_dim=768, text_dim=768, video_dim=768,
                                 output_dim1=6, output_dim2=0, dropout=0.0, hidden_dim=64, grad_clip=-1.0, seed=0)
    torch.manual_seed(0)
    model = get_models(args).cuda()
    sd = {k: v.detach().cpu().clone() for k, v in model.model.state_dict().items()}
    assert sd["fc_out_2.weight"].shape == (0, 64)
    B = 9
    xs = [K._randn((B, 768), 800 + i, cuda) for i in range(3)]
    emo, _ = K._labels(B, 6, 0, 4, cuda)
    feats, eo, vo, _ = model({"audios": xs[0], "texts": xs[1], "videos": xs[2]})
    assert vo.shape == (B, 0)
    loss = torch.nn.functional.cross_entropy(eo, emo, reduction="sum") / B
    loss.backward()
    ref = R.fusion_f64(sd, xs, 0.0, None, emo, _empty_vals(B, cuda))
    views = {n: p.grad for n, p in model.model.named_parameters()}
    _close_grads("emo-only-autograd", "grads", views, ref["grads"], 768, K.DEPTH_MLP)
    K._report("emo-only-autograd")


FRM = [("frm-H32-B1-hash", 32, (1, 2, 64), 1, "hash"), ("frm-H128-B300-ext", 128, (2, 64, 1), 300, "ext")]


@pytest.mark.parametrize("hidden,lens,B,masks", [pytest.param(*c[1:], id=c[0]) for c in FRM])
def test_frame_level_out2_0(cuda, request, hidden, lens, B, masks):
    from mertools_b200.fusion import FusionNet
    case = "emo-only-" + request.node.callspec.id
    widths = (64, 130, 3)
    sd = S.fusion_state_dict(seed=5, audio_dim=widths[0], text_dim=widths[1], video_dim=widths[2], hidden=hidden,
                             out2=0, feat_type="frm_align")
    xs = [K._randn((B, T, w), 400 + i, cuda) for i, (T, w) in enumerate(zip(lens, widths))]
    emo, _ = K._labels(B, 6, 0, 7, cuda)
    val = _empty_vals(B, cuda)
    mw = [hidden] * 3 + [3 * hidden]
    km = K._hash_masks(SEED, 0, B, mw, cuda) if masks == "hash" else K._ext_masks(B, mw, cuda)
    ref = R.fusion_f64(sd, xs, P, km, emo, val)
    n = FusionNet(*widths, hidden, 6, 0, dropout=P, device=cuda, max_batch=B, seed=SEED, feat_type="frm_align")
    n.load_state_dict(sd)
    p0 = n.params.clone()
    loss, eo, vo = n.train_step(*xs, emo, val, lr=LR, weight_decay=WD, ext_masks=km if masks == "ext" else None,
                                use_graph=False)
    Kmax = max(max(widths), 4 * hidden, B * max(lens))
    depth = K.DEPTH_MLP + 2 * max(lens)
    assert vo.shape == (B, 0) and float(loss[1]) == 0.0 and float(loss[2]) == float(loss[0])
    K._close(case, "loss total", loss[2:3], torch.tensor([ref["loss"][2]]), abs(ref["loss"][2]), Kmax, depth // 2)
    K._close(case, "emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), Kmax, depth // 2)
    _close_grads(case, "fwd_bwd", n.named_views(n.grads), ref["grads"], Kmax, depth)
    K._adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, 1)
    f2, e2, v2, _ = n.train(False).forward({"audios": xs[0], "texts": xs[1], "videos": xs[2]})
    assert v2.shape == (B, 0)
    K._report(case)


TOPN = [  # id, widths, hidden, B, masks, clip
    ("topn-N1-H4", [6373], 4, 7, "hash", -1.0),
    ("topn-N3-H64-ext", [96, 3, 128], 64, 33, "ext", -1.0),
    ("topn-N6-H128-clip", [96, 128, 768, 1024, 64, 100], 128, 32, "hash", 0.01),
    ("topn-N18-H256", [1, 3, 4096, 6373, 3, 1] * 3, 256, 20, "hash", -1.0),
]


@pytest.mark.parametrize("widths,hidden,B,masks,clip", [pytest.param(*c[1:], id=c[0]) for c in TOPN])
def test_topn_out2_0(cuda, request, widths, hidden, B, masks, clip):
    from mertools_b200.fusion import TopnFusionNet
    case = "emo-only-" + request.node.callspec.id
    N = len(widths)
    sd = S.fusion_topn_state_dict(widths, seed=8, hidden=hidden, out2=0)
    xs = [K._randn((B, w), 500 + i, cuda) for i, w in enumerate(widths)]
    emo, _ = K._labels(B, 6, 0, 8, cuda)
    val = _empty_vals(B, cuda)
    mw = list(widths) + [N * hidden]
    km = K._hash_masks(SEED, 0, B, mw, cuda) if masks == "hash" else K._ext_masks(B, mw, cuda)
    ref = R.fusion_f64(sd, xs, P, km, emo, val)
    n = TopnFusionNet(widths, hidden, 6, 0, dropout=P, grad_clip=clip, device=cuda, seed=SEED).load_state_dict(sd)
    p0 = n.params.clone()
    loss, eo, vo = n.train_step(xs, emo, val, lr=LR, weight_decay=WD, ext_masks=km if masks == "ext" else None)
    Kmax = max(max(widths), N * hidden, B)
    assert vo.shape == (B, 0)
    _check_losses(case, "topn_step", loss, ref, Kmax)
    K._close(case, "emos", eo, ref["out"][1], float(ref["out"][1].abs().max()), Kmax, K.DEPTH_MLP // 2)
    _close_grads(case, "topn_step", n.named_views(n.grads), ref["grads"], Kmax, K.DEPTH_MLP)
    K._adam_close(case, n.params, p0, n.grads, n.exp_avg, n.exp_avg_sq, 1, clip=clip if clip != -1 else 0.0)
    # eval forward with a NULL vals_out
    f, e, v, _ = n.train(False).forward({f"feat{i}": x for i, x in enumerate(xs)})
    ref_e = R.fusion_f64(n.state_dict(), xs)["out"][1]
    K._close(case, "eval emos", e, ref_e, float(ref_e.abs().max()), Kmax, K.DEPTH_MLP // 2)
    K._report(case)


# ---- NULL vals / vals_out -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out2", [0, 1])
def test_null_vals_only_at_out2_0(cuda, out2):
    """mer_fusion_forward / _fwd_bwd / _step, the frame-level forward and fwd_bwd and the top-N step take NULL vals and
    vals_out when out2 == 0 and refuse them when out2 >= 1."""
    import ctypes as C

    from mertools_b200 import _lib as L
    from mertools_b200.fusion import FusionNet, MerAdamHyper, TopnFusionNet
    B, H = 5, 64
    ok = out2 == 0
    x = [K._randn((B, 96), 900 + i, cuda) for i in range(3)]
    emo, _ = K._labels(B, 6, 1, 3, cuda)
    feats, emos = torch.empty(B, H, device=cuda), torch.empty(B, 6, device=cuda)
    st = L.stream_ptr()
    rcs = {}
    n = FusionNet(96, 96, 96, H, 6, out2, device=cuda, max_batch=B)
    d = C.byref(n.dims)
    rcs["forward"] = n._fwd(d, L.ptr(n.params), *map(L.ptr, x), B, L.ptr(n.ws), n.ws.numel(), L.ptr(feats),
                            L.ptr(emos), None, st)
    rcs["fwd_bwd"] = n._fb(d, L.ptr(n.params), L.ptr(n.grads), *map(L.ptr, x), L.ptr(emo), None, B, 1.0 / B, 0.0, 0,
                           L.ptr(n.step_counter), None, L.ptr(n.ws), n.ws.numel(), L.ptr(n.loss), L.ptr(feats),
                           L.ptr(emos), None, st)
    hyper = MerAdamHyper(1e-3, 0.9, 0.999, 1e-8, 0.0, 0.0)
    rcs["step"] = n._step(d, L.ptr(n.params), L.ptr(n.grads), L.ptr(n.exp_avg), L.ptr(n.exp_avg_sq), *map(L.ptr, x),
                          L.ptr(emo), None, B, 1.0 / B, 0.0, 0, L.ptr(n.step_counter), None, C.byref(hyper),
                          L.ptr(n.ws), n.ws.numel(), L.ptr(n.loss), L.ptr(feats), L.ptr(emos), None, st)
    nf = FusionNet(96, 96, 96, H, 6, out2, device=cuda, max_batch=B, feat_type="frm_align")
    xf = [t.view(B, 1, 96) for t in x]
    ws = nf._frm_ws(B, *xf)
    df = C.byref(nf.dims)
    rcs["frm_forward"] = nf._fwd_frm(df, L.ptr(nf.params), *map(L.ptr, xf), 1, 1, 1, B, L.ptr(ws), ws.numel(),
                                     L.ptr(feats), L.ptr(emos), None, st)
    rcs["frm_fwd_bwd"] = nf._fb_frm(df, L.ptr(nf.params), L.ptr(nf.grads), *map(L.ptr, xf), 1, 1, 1, L.ptr(emo), None,
                                    B, 1.0 / B, 0.0, 0, L.ptr(nf.step_counter), None, L.ptr(ws), ws.numel(),
                                    L.ptr(nf.loss), L.ptr(feats), L.ptr(emos), None, st)
    nt = TopnFusionNet([96, 96], H, 6, out2, device=cuda)
    need = int(L.lib().mer_fusion_topn_workspace_bytes(C.byref(nt.dims), B))
    wt = torch.empty(need, dtype=torch.uint8, device=cuda)
    fp = (C.c_void_p * 2)(x[0].data_ptr(), x[1].data_ptr())
    for name, e in (("topn_eval", None), ("topn_train", emo)):
        rcs[name] = nt._step(C.byref(nt.dims), L.ptr(nt.params), L.ptr(nt.grads), C.cast(fp, C.c_void_p), L.ptr(e),
                             None, B, 1.0 / B, 0.0, 0, L.ptr(nt.step_counter), None, L.ptr(wt), wt.numel(),
                             L.ptr(nt.loss), L.ptr(feats), L.ptr(emos), None, st)
    torch.cuda.synchronize()
    print(f"[emo-only] out2 {out2}: return codes {rcs}")
    for name, rc in rcs.items():
        assert (rc == 0) == ok, f"{name}: return code {rc} at out2 = {out2}"


# ---- the CLI against the golden of the unmodified MER2026 trainer --------------------------------------------------------
@pytest.mark.parametrize("cfg_name", ["attention", "topn2_avt", "topn2_at"])
def test_main_release_mer2026_reproduces_the_unmodified_reference_run(cuda, tmp_path, cfg_name):
    """tests/golden/main_release_mer2026_golden.npz holds ``runpy`` of the UNMODIFIED MER2026_Track1/main-release.py
    (make_golden_main_release_mer2026.py: 80 + 20 clips, 5 folds x 3 epochs, dropout 0, seeded with 0).  Same fold
    split and sample order, same best epochs, losses within 1e-3 relative, the same result-file names."""
    from mertools_b200 import main_release as MR
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "main_release_mer2026_golden.npz"))
    pre = f"{cfg_name}_"
    label_path, feats = S.write_mer2026_corpus(str(tmp_path), seed=int(g["seed"]))
    cfg = types.SimpleNamespace(PATH_TO_LABEL={"MER2026": label_path}, PATH_TO_FEATURES={"MER2026": feats})
    hyper = tmp_path / "hyper.yaml"
    hyper.write_text(str(g["hyper"]))
    argv = {"attention": ["--model=attention"] + [f"--{m}_feature=chinese-hubert-base-UTT"
                                                  for m in ("audio", "text", "video")],
            "topn2_avt": ["--model=attention_topn", "--fusion_topn=2", "--fusion_modality=AVT"],
            "topn2_at": ["--model=attention_topn", "--fusion_topn=2", "--fusion_modality=AT"]}[cfg_name]
    args = MR.build_parser().parse_args(["--dataset=MER2026", *argv, f"--hyper_path={hyper}",
                                         f"--epochs={int(g['epochs'])}", f"--save_root={tmp_path}/saved", "--gpu=0"])
    torch.manual_seed(int(g["seed"]))
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    log = {}
    saved = MR.main(args, config=cfg, log=log)
    E = int(g["epochs"])
    for f in range(5):
        assert log["eval_names"][f * E] == list(g[f"{pre}fold{f}_eval_names_epoch0"]), f"fold {f}: eval split / order"
        assert log["train_names"][f * E] == list(g[f"{pre}fold{f}_train_names_epoch0"]), f"fold {f}: train order"
    assert log["best_index"] == list(g[pre + "best_index"])
    rel = lambda a, b: np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max()  # noqa: E731
    tr, ev = np.array(log["train_loss"]).reshape(5, E), np.array(log["eval_loss"]).reshape(5, E)
    ts = np.array(log["test_loss"]).reshape(5, E, 1).transpose(2, 0, 1)
    print(f"main-release MER2026 golden {cfg_name}: train loss rel {rel(tr, g[pre + 'train_loss']):.2e}, "
          f"eval {rel(ev, g[pre + 'eval_loss']):.2e}, test {rel(ts, g[pre + 'test_loss']):.2e}")
    assert rel(tr, g[pre + "train_loss"]) < 1e-3 and rel(ev, g[pre + "eval_loss"]) < 1e-3
    assert rel(ts, g[pre + "test_loss"]) < 1e-3
    for f, best in enumerate(log["folder_save"]):
        assert best["eval_names"] == list(g[f"{pre}fold{f}_eval_names"])
        for k in ("eval_emoprobs", "test1_emoprobs"):
            assert rel(best[k], g[f"{pre}fold{f}_{k}"]) < 1e-3, (f, k)
        assert "eval_valmse" not in best
    assert len(saved) == 2
    for path, ref in zip(saved, g[pre + "saved"]):
        assert os.path.basename(path).rsplit("_", 1)[0] == str(ref)
    stored = np.load(saved[1], allow_pickle=True)
    assert stored["emo_probs"].shape == (20, 6)
    assert "-multitop-others" in saved[0] if cfg_name != "attention" else "-unimodal" in saved[0]


# ---- top-N under data parallelism -----------------------------------------------------------------------------------------
DP_WIDTHS = [96, 128, 64, 100, 40, 128]
DP_BATCHES = (27, 5)   # a 27-row batch splits 14 / 13 over two ranks; then a last batch of 5 (3 / 2)


def _dp_worker(rank, world, port, backend, out):
    import torch.distributed as dist

    from mertools_b200.fusion import TopnFusionNet
    dev = torch.device("cuda", rank if torch.cuda.device_count() >= world else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    sd = S.fusion_topn_state_dict(DP_WIDTHS, seed=8, hidden=64, out2=0)
    batches = []
    for i, n in enumerate(DP_BATCHES):
        xs = [K._randn((n, w), 1000 + 10 * i + j, dev) for j, w in enumerate(DP_WIDTHS)]
        emo, _ = K._labels(n, 6, 0, 20 + i, dev)
        batches.append((xs, emo, _empty_vals(n, dev)))
    net = TopnFusionNet(DP_WIDTHS, 64, 6, 0, dropout=0.0, device=dev)
    if rank == 0:
        net.load_state_dict(sd)
    net.broadcast_from(0)                      # rank 1 starts from zeros: the broadcast makes it a replica
    losses = []
    for _ in range(2):
        for xs, emo, val in batches:
            mine = [x[rank::world].contiguous() for x in xs]
            loss, _, _ = net.train_step(mine, emo[rank::world].contiguous(), val[rank::world].contiguous(), lr=1e-3,
                                        weight_decay=1e-5, world_size=world, global_batch=len(emo))
            losses.append(loss.clone())
    torch.cuda.synchronize()
    sig = torch.stack([net.params.double().sum(), net.params.double().abs().sum()])
    lo, hi = sig.clone(), sig.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    if rank == 0:
        ref = TopnFusionNet(DP_WIDTHS, 64, 6, 0, dropout=0.0, device=dev).load_state_dict(sd)
        ref_losses = []
        for _ in range(2):
            for xs, emo, val in batches:
                l, _, _ = ref.train_step(xs, emo, val, lr=1e-3, weight_decay=1e-5)
                ref_losses.append(l.clone())
        out["loss_diff"] = max(float((x - y).abs().max()) for x, y in zip(losses, ref_losses))
        out["loss0"] = float(ref_losses[0][2])
        out["param_rel"] = float((net.params - ref.params).norm() / ref.params.norm())
        out["same_replicas"] = bool(torch.equal(lo, hi))
    if rank == 1:
        net.params[0] += 1.0
    net._replicas_checked = False
    try:
        net.check_replicas(world)
        caught = False
    except RuntimeError:
        caught = True
    out[f"caught{rank}"] = caught
    dist.destroy_process_group()


def test_topn_two_ranks_equal_one_rank_on_the_concatenated_batch(cuda):
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
    print(f"data-parallel top-N fusion ({backend}): {out}")
    assert out["same_replicas"] and out["caught0"] and out["caught1"]
    assert out["loss_diff"] <= 1e-5 * max(1.0, out["loss0"]) and out["param_rel"] <= 1e-5
