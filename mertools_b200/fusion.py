"""Attention-fusion training on the device — mirror of MERBench ``toolkit/models`` (get_models,
Attention), ``toolkit/utils/loss.py`` and the step of ``main-release.py:train_or_eval_model``.

``FusionNet`` owns flat fp32 parameter / gradient / Adam-moment buffers (reference state_dict order)
and drives libmer_b200.so: eval forward, or one fused training step = forward + CELoss + MSELoss +
backward + Adam in two kernels (csrc/fusion_fused.cu), replayed as a CUDA graph; under data parallelism the
gradient (with the three loss scalars riding behind it) takes one NCCL all-reduce between the backward and the
Adam kernel.

``get_models(args)`` is the reference's object (toolkit/models/__init__.py:18-46): a ``torch.nn.Module`` whose
``.model`` is the Attention net, whose ``parameters()`` are ``nn.Parameter`` views of the flat buffer under the
reference's names, and whose forward is an autograd node over the same two kernels -- so the reference's own
``train_or_eval_model`` (forward, ``cls_loss + reg_loss``, ``loss.backward()``, ``clip_grad_value_``,
``torch.optim.Adam.step()``, main-release.py:17-87) runs on it unchanged.  ``train_or_eval_model`` here is that
loop; handed this module's ``Adam`` holder instead of ``torch.optim.Adam`` it takes the fused step.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L

ENC = ("audio_encoder", "text_encoder", "video_encoder", "attention_mlp")


class MerFusionDims(C.Structure):
    _fields_ = [("audio_dim", C.c_int), ("text_dim", C.c_int), ("video_dim", C.c_int),
                ("hidden", C.c_int), ("out1", C.c_int), ("out2", C.c_int)]


class MerAdamHyper(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("lr", "beta1", "beta2", "eps", "weight_decay", "grad_clip")]


LSTM_PARAMS = ("rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0",
               "linear_1.weight", "linear_1.bias")


_M64 = (1 << 64) - 1


def rank_dropout_seed(seed, rank, world_size):
    """The dropout seed one data-parallel rank hands the kernels.  The keep-masks hash (seed, mask tensor, step, LOCAL
    element index), so ranks that share a seed would drop the same elements of their local rows, and the all-reduced
    gradient would carry W-fold correlated dropout noise.  At world_size 1 the seed is returned unchanged; otherwise it
    is a splitmix64 output for (seed, rank): a bijection of the seed for each rank, different for every rank."""
    seed = int(seed) & _M64
    if world_size == 1:
        return seed
    z = (seed + 0x9E3779B97F4A7C15 * (int(rank) + 1)) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def _dist_seed(seed, world):
    if world == 1:
        return seed
    import torch.distributed as dist
    return rank_dropout_seed(seed, dist.get_rank(), world)


def param_names(feat_type="utt"):
    names = []
    for e in ENC:
        if feat_type != "utt" and e != "attention_mlp":  # LSTMEncoder (encoder.py:45-72)
            names += [f"{e}.{n}" for n in LSTM_PARAMS]
            continue
        for l in ("linear_1", "linear_2", "linear_3"):
            names += [f"{e}.{l}.weight", f"{e}.{l}.bias"]
    for l in ("fc_att", "fc_out_1", "fc_out_2"):
        names += [f"{l}.weight", f"{l}.bias"]
    return names


def param_shapes(audio_dim, text_dim, video_dim, hidden, out1, out2, feat_type="utt"):
    ins = dict(audio_encoder=audio_dim, text_encoder=text_dim, video_encoder=video_dim,
               attention_mlp=3 * hidden)
    shapes = {}
    for e in ENC:
        if feat_type != "utt" and e != "attention_mlp":
            shapes[f"{e}.rnn.weight_ih_l0"] = (4 * hidden, ins[e])
            shapes[f"{e}.rnn.weight_hh_l0"] = (4 * hidden, hidden)
            shapes[f"{e}.rnn.bias_ih_l0"] = (4 * hidden,)
            shapes[f"{e}.rnn.bias_hh_l0"] = (4 * hidden,)
            shapes[f"{e}.linear_1.weight"] = (hidden, hidden)
            shapes[f"{e}.linear_1.bias"] = (hidden,)
            continue
        shapes[f"{e}.linear_1.weight"] = (hidden, ins[e])
        shapes[f"{e}.linear_1.bias"] = (hidden,)
        for l in ("linear_2", "linear_3"):
            shapes[f"{e}.{l}.weight"] = (hidden, hidden)
            shapes[f"{e}.{l}.bias"] = (hidden,)
    for l, o in (("fc_att", 3), ("fc_out_1", out1), ("fc_out_2", out2)):
        shapes[f"{l}.weight"] = (o, hidden)
        shapes[f"{l}.bias"] = (o,)
    return shapes


class FusionNet:
    """Device-resident Attention fusion model.  feat_type 'utt': MLP encoders on [B, D] features;
    'frm_align' / 'frm_unalign': LSTM encoders on [B, T, D] sequences (attention.py:25-33)."""

    def __init__(self, audio_dim=768, text_dim=768, video_dim=768, hidden_dim=128, output_dim1=6,
                 output_dim2=1, dropout=0.0, grad_clip=-1.0, device="cuda", max_batch=4096, seed=0,
                 feat_type="utt"):
        L.check(L.lib().mer_check_device())
        assert feat_type in ("utt", "frm_align", "frm_unalign"), feat_type
        self.feat_type = feat_type
        self.frm = feat_type != "utt"
        self.device = torch.device(device)
        self.dims = MerFusionDims(audio_dim, text_dim, video_dim, hidden_dim, output_dim1, output_dim2)
        self.dropout, self.grad_clip, self.seed = float(dropout), float(grad_clip), int(seed)
        lib = L.lib()
        lib.mer_fusion_param_count.restype = C.c_longlong
        lib.mer_fusion_param_count.argtypes = [C.POINTER(MerFusionDims)]
        lib.mer_fusion_workspace_bytes.restype = C.c_longlong
        lib.mer_fusion_workspace_bytes.argtypes = [C.POINTER(MerFusionDims), C.c_int]
        vp, i32, f32, i64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong
        self._fwd = L.declare("mer_fusion_forward", [C.POINTER(MerFusionDims), vp, vp, vp, vp, i32, vp,
                                                     i64, vp, vp, vp, vp])
        self._fb = L.declare("mer_fusion_fwd_bwd", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, vp, vp,
                                                    i32, f32, f32, C.c_ulonglong, vp, vp, vp, i64, vp,
                                                    vp, vp, vp, vp])
        self._adam = L.declare("mer_fusion_adam", [vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, f32,
                                                   f32, vp, vp])
        self._step = L.declare("mer_fusion_step", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                                   i32, f32, f32, C.c_ulonglong, vp, vp, C.POINTER(MerAdamHyper),
                                                   vp, i64, vp, vp, vp, vp, vp])
        self._fwd_train = L.declare("mer_fusion_forward_train", [C.POINTER(MerFusionDims), vp, vp, vp, vp, i32, f32,
                                                                 C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp])
        self._bwd = L.declare("mer_fusion_backward", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp, i32, vp, vp, vp,
                                                      f32, C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp])
        if self.frm:
            lib.mer_fusion_frm_param_count.restype = C.c_longlong
            lib.mer_fusion_frm_param_count.argtypes = [C.POINTER(MerFusionDims)]
            lib.mer_fusion_frm_workspace_bytes.restype = C.c_longlong
            lib.mer_fusion_frm_workspace_bytes.argtypes = [C.POINTER(MerFusionDims)] + [i32] * 4
            self._fwd_frm = L.declare("mer_fusion_frm_forward", [C.POINTER(MerFusionDims), vp, vp, vp, vp, i32,
                                                                 i32, i32, i32, vp, i64, vp, vp, vp, vp])
            self._fb_frm = L.declare("mer_fusion_frm_fwd_bwd", [C.POINTER(MerFusionDims), vp, vp, vp, vp, vp,
                                                                i32, i32, i32, vp, vp, i32, f32, f32,
                                                                C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp,
                                                                vp])
        self.n_params = int((lib.mer_fusion_frm_param_count if self.frm else lib.mer_fusion_param_count)(
            C.byref(self.dims)))
        self.shapes = param_shapes(audio_dim, text_dim, video_dim, hidden_dim, output_dim1, output_dim2,
                                   feat_type)
        assert sum(int(np.prod(s)) for s in self.shapes.values()) == self.n_params
        z = lambda: torch.zeros(self.n_params, dtype=torch.float32, device=self.device)  # noqa: E731
        self.params, self.exp_avg, self.exp_avg_sq = z(), z(), z()
        # the gradient and the three loss scalars share one allocation: ONE all-reduce under data parallelism
        self._grads_loss = torch.zeros(self.n_params + 4, dtype=torch.float32, device=self.device)
        self.grads = self._grads_loss[:self.n_params]
        self.loss = self._grads_loss[self.n_params:self.n_params + 3]
        self.step_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.max_batch = max_batch
        self.ws = torch.empty(int(lib.mer_fusion_workspace_bytes(C.byref(self.dims), max_batch)) if not self.frm
                              else 0, dtype=torch.uint8, device=self.device)
        self.training = True
        self.graph_launches = 0  # kernels launched through CUDA-graph replays (not seen by the library counter)
        lib.mer_launch_count.restype = C.c_longlong
        self._graphs = {}
        self._static = None

    # ---- nn.Module-flavoured surface used by the reference loop --------------------------------
    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def cuda(self):
        return self

    def parameters(self):
        return [self.params]

    def named_views(self, flat=None):
        flat = self.params if flat is None else flat
        out, o = {}, 0
        for n in param_names(self.feat_type):
            k = int(np.prod(self.shapes[n]))
            out[n] = flat[o:o + k].view(self.shapes[n])
            o += k
        return out

    def state_dict(self):
        return {k: v.clone() for k, v in self.named_views().items()}

    def load_state_dict(self, sd):
        """Accepts the reference's names with or without the ``model.`` wrapper prefix
        (toolkit/models/__init__.py wraps the net as ``.model``)."""
        views = self.named_views()
        for n, dst in views.items():
            src = sd[n] if n in sd else sd["model." + n]
            if isinstance(src, np.ndarray):
                src = torch.from_numpy(src)
            dst.copy_(src.to(self.device, torch.float32))
        self._invalidate()
        return self

    def _invalidate(self):
        self._graphs.clear()

    # ---- forward / step --------------------------------------------------------------------------
    def _bufs(self, B):
        d = self.dims
        f = lambda n: torch.empty(B, n, dtype=torch.float32, device=self.device)  # noqa: E731
        return f(d.hidden), f(d.out1), f(d.out2)

    def forward(self, batch):
        """batch: dict with 'audios','texts','videos' fp32 CUDA [B,D].  Eval-mode forward; returns
        (features, emos_out, vals_out, interloss) like Attention.forward (attention.py:36-57)."""
        a, t, v = (batch[k].contiguous() for k in ("audios", "texts", "videos"))
        B = a.shape[0]
        assert B <= self.max_batch
        feats, emos, vals = self._bufs(B)
        if self.frm:
            ws = self._frm_ws(B, a, t, v)
            L.check(self._fwd_frm(C.byref(self.dims), L.ptr(self.params), L.ptr(a), L.ptr(t), L.ptr(v),
                                  a.shape[1], t.shape[1], v.shape[1], B, L.ptr(ws), ws.numel(), L.ptr(feats),
                                  L.ptr(emos), L.ptr(vals), L.stream_ptr()))
            return feats, emos, vals, torch.zeros((), dtype=torch.int64, device=self.device)
        L.check(self._fwd(C.byref(self.dims), L.ptr(self.params), L.ptr(a), L.ptr(t), L.ptr(v), B,
                          L.ptr(self.ws), self.ws.numel(), L.ptr(feats), L.ptr(emos), L.ptr(vals),
                          L.stream_ptr()))
        return feats, emos, vals, torch.zeros((), dtype=torch.int64, device=self.device)

    __call__ = forward

    def _frm_ws(self, B, a, t, v):
        """Workspace of the frame-level variant: depends on the three padded sequence lengths."""
        assert a.dim() == t.dim() == v.dim() == 3, "frame-level features are [B, T, D] (read_data.py:118-125)"
        need = int(L.lib().mer_fusion_frm_workspace_bytes(C.byref(self.dims), B, a.shape[1], t.shape[1],
                                                          v.shape[1]))
        if self.ws.numel() < need:
            self.ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            self._invalidate()
        return self.ws

    def _masks(self, ext_masks):
        if ext_masks is None:
            return None
        arr = (C.c_void_p * 4)(*[m.data_ptr() if m is not None else None for m in ext_masks])
        return C.cast(arr, C.c_void_p)

    def _launch_step(self, a, t, v, emo, val, feats, emos_out, vals_out, lr, betas, eps, wd,
                     world, ext_masks, global_batch=None, fused_adam=True):
        B = a.shape[0]
        inv = 1.0 / (global_batch if global_batch is not None else B * world)
        masks = self._masks(ext_masks)
        clip = self.grad_clip if self.grad_clip != -1 else 0.0
        seed = _dist_seed(self.seed, world)
        if not self.frm and world == 1 and fused_adam:  # the whole step in two kernels, Adam fused into the weight gradients
            hyper = MerAdamHyper(lr, betas[0], betas[1], eps, wd, clip)
            L.check(self._step(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(self.exp_avg),
                               L.ptr(self.exp_avg_sq), L.ptr(a), L.ptr(t), L.ptr(v), L.ptr(emo), L.ptr(val), B,
                               inv, self.dropout, seed, L.ptr(self.step_counter), masks, C.byref(hyper),
                               L.ptr(self.ws), self.ws.numel(), L.ptr(self.loss), L.ptr(feats), L.ptr(emos_out),
                               L.ptr(vals_out), L.stream_ptr()))
            return
        if self.frm:
            ws = self._frm_ws(B, a, t, v)
            L.check(self._fb_frm(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(a), L.ptr(t),
                                 L.ptr(v), a.shape[1], t.shape[1], v.shape[1], L.ptr(emo), L.ptr(val), B,
                                 inv, self.dropout, seed, L.ptr(self.step_counter), masks,
                                 L.ptr(ws), ws.numel(), L.ptr(self.loss), L.ptr(feats), L.ptr(emos_out),
                                 L.ptr(vals_out), L.stream_ptr()))
        else:
            L.check(self._fb(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(a), L.ptr(t),
                             L.ptr(v), L.ptr(emo), L.ptr(val), B, inv, self.dropout,
                             seed, L.ptr(self.step_counter), masks, L.ptr(self.ws), self.ws.numel(),
                             L.ptr(self.loss), L.ptr(feats), L.ptr(emos_out), L.ptr(vals_out), L.stream_ptr()))
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(self._grads_loss)  # SUM: gradient and loss terms already carry 1 / global_batch
        L.check(self._adam(L.ptr(self.params), L.ptr(self.grads), L.ptr(self.exp_avg),
                           L.ptr(self.exp_avg_sq), self.n_params, lr, betas[0], betas[1], eps, wd, 1.0,
                           clip, L.ptr(self.step_counter), L.stream_ptr()))

    def train_step(self, a, t, v, emo, val, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                   world_size=1, ext_masks=None, use_graph=True, global_batch=None, fused_adam=True):
        """One optimisation step on a device batch.  Returns (loss[3] device tensor, emos_out,
        vals_out).  With use_graph the launch sequence is captured once per batch shape and replayed; inputs
        are copied into static buffers first.  world_size > 1: this rank's slice of a data-parallel batch of
        ``global_batch`` rows (default: batch * world_size); the loss returned is the global one."""
        B = a.shape[0]
        assert B <= self.max_batch and emo.dtype == torch.int64 and val.dtype == torch.float32
        if world_size > 1:
            self.check_replicas(world_size)
        # under data parallelism the step is launched eagerly (4 launches around the NCCL all-reduce)
        if not use_graph or ext_masks is not None or world_size > 1 or not fused_adam:
            feats, emos_out, vals_out = self._bufs(B)
            self._launch_step(a.contiguous(), t.contiguous(), v.contiguous(), emo.contiguous(),
                              val.contiguous(), feats, emos_out, vals_out, lr, betas, eps,
                              weight_decay, world_size, ext_masks, global_batch, fused_adam)
            return self.loss, emos_out, vals_out
        if self.frm:
            self._frm_ws(B, a, t, v)  # sized (and graphs invalidated on growth) before any capture
        key = (B, tuple(a.shape[1:]), tuple(t.shape[1:]), tuple(v.shape[1:]), lr, betas, eps, weight_decay,
               world_size, self.dropout, self.grad_clip)
        if key not in self._graphs:
            st = dict(a=torch.empty_like(a), t=torch.empty_like(t), v=torch.empty_like(v),
                      emo=torch.empty_like(emo), val=torch.empty_like(val))
            st["feats"], st["emos"], st["vals"] = self._bufs(B)
            for k, src in (("a", a), ("t", t), ("v", v), ("emo", emo), ("val", val)):
                st[k].copy_(src)
            # warm-up outside capture on a side stream, with state restored afterwards
            saved = [x.clone() for x in (self.params, self.exp_avg, self.exp_avg_sq, self.step_counter)]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._launch_step(st["a"], st["t"], st["v"], st["emo"], st["val"], st["feats"],
                                  st["emos"], st["vals"], lr, betas, eps, weight_decay, world_size, None)
            torch.cuda.current_stream().wait_stream(s)
            for dst, src in zip((self.params, self.exp_avg, self.exp_avg_sq, self.step_counter), saved):
                dst.copy_(src)
            g = torch.cuda.CUDAGraph()
            n0 = L.lib().mer_launch_count()
            with torch.cuda.graph(g):
                self._launch_step(st["a"], st["t"], st["v"], st["emo"], st["val"], st["feats"],
                                  st["emos"], st["vals"], lr, betas, eps, weight_decay, world_size, None)
            self._graphs[key] = (g, st, int(L.lib().mer_launch_count() - n0))
        g, st, n_kernels = self._graphs[key]
        for k, src in (("a", a), ("t", t), ("v", v), ("emo", emo), ("val", val)):
            st[k].copy_(src, non_blocking=True)
        g.replay()
        self.graph_launches += n_kernels
        return self.loss, st["emos"], st["vals"]


    # ---- data parallelism ------------------------------------------------------------------------
    def broadcast_from(self, src=0):
        """Make every rank a replica of rank ``src`` (parameters, Adam moments, step counter): SURVEY.md §8e
        'identical initial weights (broadcast once)'."""
        import torch.distributed as dist
        for buf in (self.params, self.exp_avg, self.exp_avg_sq, self.step_counter):
            dist.broadcast(buf, src)
        self._replicas_checked = False
        return self

    def check_replicas(self, world):
        """Once per model: the ranks must hold identical parameters, or the all-reduced gradient trains W
        different models.  One small all-reduce of (sum, sum of squares) min against max."""
        if getattr(self, "_replicas_checked", False):
            return
        import torch.distributed as dist
        sig = torch.stack([self.params.double().sum(), (self.params.double() ** 2).sum()])
        lo, hi = sig.clone(), sig.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        if not torch.equal(lo, hi):
            raise RuntimeError("FusionNet: the data-parallel ranks hold different parameters "
                               "(call broadcast_from(0) after construction / load_state_dict)")
        self._replicas_checked = True

    # ---- the two halves of the autograd node (utterance-level net) -----------------------------------
    def forward_train(self, a, t, v, ext_masks=None):
        """Train-mode forward (dropout from (seed, step_counter) or ext_masks) -> (features, emos_out, vals_out)."""
        assert not self.frm, "the autograd node covers the utterance-level Attention net"
        B = a.shape[0]
        assert B <= self.max_batch
        feats, emos, vals = self._bufs(B)
        L.check(self._fwd_train(C.byref(self.dims), L.ptr(self.params), L.ptr(a), L.ptr(t), L.ptr(v), B, self.dropout,
                                self.seed, L.ptr(self.step_counter), self._masks(ext_masks), L.ptr(self.ws),
                                self.ws.numel(), L.ptr(feats), L.ptr(emos), L.ptr(vals), L.stream_ptr()))
        return feats, emos, vals

    def backward(self, a, t, v, d_feats, d_emos, d_vals, ext_masks=None):
        """d(loss)/d(params) into ``self.grads`` from the upstream gradients of forward_train's outputs (None =
        zero); must see the same inputs, masks and step counter as the forward it differentiates."""
        B = a.shape[0]
        feats, emos, vals = self._bufs(B)
        c = lambda g: None if g is None else g.contiguous().float()  # noqa: E731
        d_feats, d_emos, d_vals = c(d_feats), c(d_emos), c(d_vals)
        L.check(self._bwd(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(a), L.ptr(t), L.ptr(v), B,
                          L.ptr(d_feats), L.ptr(d_emos), L.ptr(d_vals), self.dropout, self.seed,
                          L.ptr(self.step_counter), self._masks(ext_masks), L.ptr(self.ws), self.ws.numel(),
                          L.ptr(feats), L.ptr(emos), L.ptr(vals), L.stream_ptr()))
        return self.grads


class MerFusionTopnDims(C.Structure):
    _fields_ = [("n_feats", C.c_int), ("feat_dims", C.c_int * 18), ("hidden", C.c_int), ("out1", C.c_int),
                ("out2", C.c_int)]


class TopnFusionNet:
    """Attention_TOPN (MER2026_Track1/toolkit/models/attention_topn.py): the utterance-level fusion net over
    N <= 18 features ``batch['feat0'] .. batch['feat{N-1}']`` ([B, feat_dims[i]] each)."""

    def __init__(self, feat_dims, hidden_dim=128, output_dim1=6, output_dim2=1, dropout=0.0, grad_clip=-1.0,
                 device="cuda", seed=0):
        L.check(L.lib().mer_check_device())
        assert 1 <= len(feat_dims) <= 18
        self.device = torch.device(device)
        self.feat_dims = [int(d) for d in feat_dims]
        self.dims = MerFusionTopnDims(len(feat_dims), (C.c_int * 18)(*self.feat_dims), hidden_dim, output_dim1,
                                      output_dim2)
        self.dropout, self.grad_clip, self.seed = float(dropout), float(grad_clip), int(seed)
        lib = L.lib()
        lib.mer_fusion_topn_param_count.restype = C.c_longlong
        lib.mer_fusion_topn_param_count.argtypes = [C.POINTER(MerFusionTopnDims)]
        lib.mer_fusion_topn_workspace_bytes.restype = C.c_longlong
        lib.mer_fusion_topn_workspace_bytes.argtypes = [C.POINTER(MerFusionTopnDims), C.c_int]
        vp, i32, f32, i64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong
        self._step = L.declare("mer_fusion_topn_step", [C.POINTER(MerFusionTopnDims), vp, vp, vp, vp, vp, i32, f32, f32,
                                                        C.c_ulonglong, vp, vp, vp, i64, vp, vp, vp, vp, vp])
        self._adam = L.declare("mer_fusion_adam", [vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, f32, f32, vp, vp])
        self.n_params = int(lib.mer_fusion_topn_param_count(C.byref(self.dims)))
        self.names, self.shapes = [], {}
        H = hidden_dim
        for i, d in enumerate(self.feat_dims + [H * len(self.feat_dims)]):
            e = f"encoder{i}" if i < len(self.feat_dims) else "attention_mlp"
            for l, k in (("linear_1", d), ("linear_2", H), ("linear_3", H)):
                self.names += [f"{e}.{l}.weight", f"{e}.{l}.bias"]
                self.shapes[f"{e}.{l}.weight"], self.shapes[f"{e}.{l}.bias"] = (H, k), (H,)
        for l, o in (("fc_att", len(self.feat_dims)), ("fc_out_1", output_dim1), ("fc_out_2", output_dim2)):
            self.names += [f"{l}.weight", f"{l}.bias"]
            self.shapes[f"{l}.weight"], self.shapes[f"{l}.bias"] = (o, H), (o,)
        assert sum(int(np.prod(s)) for s in self.shapes.values()) == self.n_params
        z = lambda: torch.zeros(self.n_params, dtype=torch.float32, device=self.device)  # noqa: E731
        self.params, self.grads, self.exp_avg, self.exp_avg_sq = z(), z(), z(), z()
        self.step_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.loss = torch.zeros(3, dtype=torch.float32, device=self.device)
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.training = True

    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def named_views(self, flat=None):
        flat = self.params if flat is None else flat
        out, o = {}, 0
        for n in self.names:
            k = int(np.prod(self.shapes[n]))
            out[n] = flat[o:o + k].view(self.shapes[n])
            o += k
        return out

    def state_dict(self):
        return {k: v.clone() for k, v in self.named_views().items()}

    def load_state_dict(self, sd):
        for n, dst in self.named_views().items():
            src = sd[n] if n in sd else sd["model." + n]
            if isinstance(src, np.ndarray):
                src = torch.from_numpy(src)
            dst.copy_(src.to(self.device, torch.float32))
        return self

    def _run(self, feats, emo, val, ext_masks, world):
        B = feats[0].shape[0]
        need = int(L.lib().mer_fusion_topn_workspace_bytes(C.byref(self.dims), B))
        if self.ws.numel() < need:
            self.ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        feats = [f.contiguous() for f in feats]
        fp = (C.c_void_p * len(feats))(*[f.data_ptr() for f in feats])
        mp = None
        if ext_masks is not None:
            mp = (C.c_void_p * len(ext_masks))(*[m.data_ptr() if m is not None else None for m in ext_masks])
        d = self.dims
        out = [torch.empty(B, n, dtype=torch.float32, device=self.device) for n in (d.hidden, d.out1, d.out2)]
        L.check(self._step(C.byref(d), L.ptr(self.params), L.ptr(self.grads), C.cast(fp, C.c_void_p), L.ptr(emo),
                           L.ptr(val), B, 1.0 / (B * world), self.dropout if emo is not None else 0.0,
                           _dist_seed(self.seed, world),
                           L.ptr(self.step_counter), C.cast(mp, C.c_void_p) if mp is not None else None,
                           L.ptr(self.ws), self.ws.numel(), L.ptr(self.loss), L.ptr(out[0]), L.ptr(out[1]),
                           L.ptr(out[2]), L.stream_ptr()))
        return out

    def forward(self, batch):
        """batch: {'feat0': [B, d0], ...}; eval-mode forward -> (features, emos_out, vals_out, interloss)."""
        feats = [batch[f"feat{i}"] for i in range(len(self.feat_dims))]
        f, e, v = self._run(feats, None, None, None, 1)
        return f, e, v, torch.zeros((), dtype=torch.int64, device=self.device)

    __call__ = forward

    def train_step(self, feats, emo, val, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, world_size=1,
                   ext_masks=None):
        """One optimisation step (forward, CE + MSE, backward, optional all-reduce, Adam)."""
        assert emo.dtype == torch.int64 and val.dtype == torch.float32
        _, eo, vo = self._run(feats, emo.contiguous(), val.contiguous(), ext_masks, world_size)
        if world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(self.grads)
        L.check(self._adam(L.ptr(self.params), L.ptr(self.grads), L.ptr(self.exp_avg), L.ptr(self.exp_avg_sq),
                           self.n_params, lr, betas[0], betas[1], eps, weight_decay, 1.0,
                           self.grad_clip if self.grad_clip != -1 else 0.0, L.ptr(self.step_counter), L.stream_ptr()))
        return self.loss, eo, vo


def reference_init(feat_type, audio_dim, text_dim, video_dim, hidden, out1, out2):
    """The state_dict ``get_models(args)`` of the reference starts from: torch's own ``nn.Linear`` / ``nn.LSTM``
    constructors, called on the CPU in the order Attention.__init__ builds its sub-modules (attention.py:25-40;
    MLPEncoder: linear_1..3, encoder.py:25-27; LSTMEncoder: rnn then linear_1, encoder.py:59-61), so the values AND
    the consumption of torch's global generator are the reference's by construction."""
    nn = torch.nn
    sd = {}

    def take(prefix, mod):
        for k, v in mod.state_dict().items():
            sd[f"{prefix}.{k}"] = v

    for e, d in (("audio_encoder", audio_dim), ("text_encoder", text_dim), ("video_encoder", video_dim),
                 ("attention_mlp", 3 * hidden)):
        if feat_type != "utt" and e != "attention_mlp":
            take(f"{e}.rnn", nn.LSTM(d, hidden, num_layers=1, dropout=0.0, bidirectional=False, batch_first=True))
            take(f"{e}.linear_1", nn.Linear(hidden, hidden))
        else:
            for l, k in (("linear_1", d), ("linear_2", hidden), ("linear_3", hidden)):
                take(f"{e}.{l}", nn.Linear(k, hidden))
    for l, o in (("fc_att", 3), ("fc_out_1", out1), ("fc_out_2", out2)):
        take(l, nn.Linear(hidden, o))
    return sd


class _FusionFn(torch.autograd.Function):
    """Attention.forward as an autograd node over libmer_b200: forward = mer_fusion_forward_train, backward =
    mer_fusion_backward (recomputes the forward from the saved inputs under the same dropout masks)."""

    @staticmethod
    def forward(ctx, module, a, t, v, *params):
        net = module.net
        a, t, v = a.contiguous().float(), t.contiguous().float(), v.contiguous().float()
        ctx.module, ctx.mask_step = module, int(module._mask_step)
        net.step_counter.fill_(ctx.mask_step)
        ctx.save_for_backward(a, t, v)
        out = net.forward_train(a, t, v)
        module._mask_step += 1
        return out

    @staticmethod
    def backward(ctx, d_feats, d_emos, d_vals):
        module, net = ctx.module, ctx.module.net
        a, t, v = ctx.saved_tensors
        net.step_counter.fill_(ctx.mask_step)
        flat = net.backward(a, t, v, d_feats, d_emos, d_vals).clone()  # autograd may keep / accumulate into these
        grads = tuple(net.named_views(flat).values())
        return (None, None, None, None) + grads


class _ParamGroup(torch.nn.Module):
    """A name-space node (``audio_encoder``, ``linear_1``, ``rnn`` ...) so that state_dict keys are the reference's."""


class Attention(torch.nn.Module):
    """toolkit/models/attention.py:8-57 on the device: same constructor argument (``args``), same parameter names,
    same ``forward(batch) -> (features, emos_out, vals_out, interloss)``.  Parameters are views of one flat buffer
    (``self.net.params``); with autograd enabled the forward is one differentiable node, otherwise the eval /
    train-mode kernels run directly.  Dropout masks come from a counter hash, not from torch's generator."""

    def __init__(self, args):
        super().__init__()
        self.grad_clip = args.grad_clip
        feat_type = getattr(args, "feat_type", "utt")
        dev = getattr(args, "device", None) or torch.device("cuda", torch.cuda.current_device())
        net = FusionNet(args.audio_dim, args.text_dim, args.video_dim, args.hidden_dim, args.output_dim1,
                        args.output_dim2, dropout=args.dropout, grad_clip=args.grad_clip, device=dev,
                        seed=getattr(args, "seed", 0), feat_type=feat_type)
        net.load_state_dict(reference_init(feat_type, args.audio_dim, args.text_dim, args.video_dim, args.hidden_dim,
                                           args.output_dim1, args.output_dim2))
        object.__setattr__(self, "net", net)  # not a sub-module: its buffers are exposed as the parameters below
        self._mask_step = 0
        self._param_order = []
        for name, view in net.named_views().items():
            node, parts = self, name.split(".")
            for part in parts[:-1]:
                if not hasattr(node, part):
                    node.add_module(part, _ParamGroup())
                node = getattr(node, part)
            prm = torch.nn.Parameter(view, requires_grad=True)
            node.register_parameter(parts[-1], prm)
            self._param_order.append(prm)

    def _apply(self, fn, recurse=True):
        """.cuda() / .to(device) are no-ops on a module that already lives on its GPU; anything that would move or
        re-type the parameters would detach them from the flat buffer the kernels read."""
        probe = fn(self._param_order[0].data)
        if probe.data_ptr() != self._param_order[0].data_ptr():
            raise RuntimeError("mertools_b200 Attention lives on its GPU in fp32; it cannot be moved or cast")
        return self

    def train(self, mode=True):
        self.net.train(mode)
        return super().train(mode)

    def forward(self, batch):
        a, t, v = batch["audios"], batch["texts"], batch["videos"]
        interloss = torch.tensor(0).cuda()  # attention.py:55
        if self.net.frm or not (torch.is_grad_enabled() and self.training):
            if self.training and not self.net.frm:
                self.net.step_counter.fill_(self._mask_step)
                self._mask_step += 1
                return (*self.net.forward_train(a.contiguous().float(), t.contiguous().float(),
                                                v.contiguous().float()), interloss)
            return (*self.net.forward(batch)[:3], interloss)
        feats, emos, vals = _FusionFn.apply(self, a, t, v, *self._param_order)
        return feats, emos, vals, interloss


class get_models(torch.nn.Module):  # noqa: N801 -- the reference's name (toolkit/models/__init__.py:18)
    """args: .model ('attention' | 'attention_topn'), .feat_type, .audio_dim/.text_dim/.video_dim, .output_dim1/
    .output_dim2, .dropout, .hidden_dim, .grad_clip.  ``.model`` is the net, ``forward(batch)`` its 4-tuple,
    ``parameters()`` feed ``torch.optim.Adam`` as in main-release.py:205."""

    def __init__(self, args):
        super().__init__()
        if args.model == "attention_topn":  # MER2026 toolkit: args.audio_dim holds the list of feature widths
            net = TopnFusionNet(args.audio_dim, args.hidden_dim, args.output_dim1, args.output_dim2,
                                dropout=args.dropout, grad_clip=args.grad_clip,
                                device=getattr(args, "device", "cuda"))
            object.__setattr__(self, "model", net)
            return
        assert args.model == "attention", "only the Attention / Attention_TOPN fusion nets are on the H100 path"
        self.model = Attention(args)

    def forward(self, batch):
        return self.model(batch)

    def train(self, mode=True):
        self.model.train(mode)
        return super().train(mode)

    def __getattr__(self, k):  # .net / .train_step / ... of the device object, for callers of the fused path
        try:
            return super().__getattr__(k)
        except AttributeError:
            if k.startswith("_"):
                raise
            model = self.__dict__.get("model") or self.__dict__.get("_modules", {}).get("model")
            if model is None:
                raise
            if hasattr(model, k):
                return getattr(model, k)
            return getattr(getattr(model, "net", model), k)


class Adam:
    """Hyper-parameter holder for the fused step: stands where ``optim.Adam(model.parameters(), lr, weight_decay)``
    stands in main-release.py:205 when the caller wants forward + losses + backward + update in two kernels
    (the update then runs inside FusionNet.train_step).  ``torch.optim.Adam`` itself works too (see get_models)."""

    def __init__(self, params=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay

    def zero_grad(self):
        pass


def mer2023_calculate_results(emo_probs=(), emo_labels=(), val_preds=(), val_labels=()):
    """toolkit/dataloader/mer2023.py:137-155."""
    from sklearn.metrics import accuracy_score, f1_score, mean_squared_error
    emo_preds = np.argmax(emo_probs, 1)
    acc = accuracy_score(emo_labels, emo_preds)
    f1 = f1_score(emo_labels, emo_preds, average="weighted")
    mse = mean_squared_error(val_labels, val_preds)
    res = dict(emoprobs=emo_probs, emolabels=emo_labels, emoacc=acc, emofscore=f1, valpreds=val_preds,
               vallabels=val_labels, valmse=mse)
    return res, f"f1:{f1:.4f}_acc:{acc:.4f}_val:{mse:.4f}"


def train_or_eval_model(args, model, reg_loss, cls_loss, dataloader, epoch, optimizer=None, train=False,
                        calculate_results=None, world_size=1):
    """main-release.py:17-87: same arguments, same ``save_results`` dict (names, loss, then the keys of
    ``dataloader_class.calculate_results``; default: the MER2023 rule).  With a ``torch.optim`` optimizer this IS the
    reference loop (zero_grad, forward, ``cls_loss + reg_loss``, backward, clip_grad_value_, step) running on the
    autograd node; with this module's ``Adam`` holder each training batch is one fused FusionNet.train_step."""
    vidnames, val_preds, val_labels, emo_probs, emo_labels, losses = [], [], [], [], [], []
    assert not train or optimizer is not None
    fused = train and isinstance(optimizer, Adam)
    net = getattr(model, "net", None) or getattr(getattr(model, "model", None), "net", None) or \
        getattr(model, "model", model)
    model.train() if train else model.eval()
    for data in dataloader:
        if train:
            optimizer.zero_grad()
        batch, emos, vals, bnames = data
        vidnames += bnames
        for key in batch:
            batch[key] = batch[key].cuda()
        emos, vals = emos.cuda(), vals.cuda()
        if fused:
            loss3, emos_out, vals_out = net.train_step(
                batch["audios"], batch["texts"], batch["videos"], emos.long(), vals.float().view(-1, 1),
                lr=optimizer.lr, betas=optimizer.betas, eps=optimizer.eps,
                weight_decay=optimizer.weight_decay, world_size=world_size)
            loss = loss3[2]
        else:
            _, emos_out, vals_out, interloss = model(batch)
            loss = interloss + cls_loss(emos_out, emos) + reg_loss(vals_out, vals)
        emo_probs.append(emos_out.data.cpu().numpy())
        emo_labels.append(emos.data.cpu().numpy())
        val_preds.append(vals_out.data.cpu().numpy())
        val_labels.append(vals.data.cpu().numpy())
        losses.append(loss.data.cpu().numpy())
        if train and not fused:
            loss.backward()
            clip = getattr(getattr(model, "model", model), "grad_clip", -1)
            if clip != -1:
                torch.nn.utils.clip_grad_value_([p for p in model.parameters() if p.requires_grad], clip)
            optimizer.step()
    emo_probs, emo_labels = np.concatenate(emo_probs), np.concatenate(emo_labels)
    val_preds, val_labels = np.concatenate(val_preds), np.concatenate(val_labels)
    results, _ = (calculate_results or mer2023_calculate_results)(emo_probs, emo_labels, val_preds, val_labels)
    return dict(names=vidnames, loss=np.mean(losses), **results)


class CELoss(torch.nn.Module):
    """toolkit/utils/loss.py:5-15 (host-side torch; used for eval-loss reporting)."""

    def forward(self, pred, target):
        pred = torch.nn.functional.log_softmax(pred, 1)
        return torch.nn.functional.nll_loss(pred, target.long(), reduction="sum") / len(pred)


class MSELoss(torch.nn.Module):
    """toolkit/utils/loss.py:18-28."""

    def forward(self, pred, target):
        pred, target = pred.view(-1, 1), target.view(-1, 1)
        return torch.nn.functional.mse_loss(pred, target, reduction="sum") / len(pred)
