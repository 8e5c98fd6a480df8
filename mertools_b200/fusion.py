"""Attention-fusion training on the device — mirror of MERBench ``toolkit/models`` (get_models,
Attention), ``toolkit/utils/loss.py`` and the step of ``main-release.py:train_or_eval_model``.

``FusionNet`` owns flat fp32 parameter / gradient / Adam-moment buffers (reference state_dict order; the
``_DeviceNet`` base it shares with ``TopnFusionNet`` and ``fusion_mlp.MlpFusionNet``) and drives libmer_b200.so: eval
forward, or one fused training step = forward + CELoss + MSELoss + backward + Adam in two kernels
(csrc/fusion_fused.cu), replayed as a CUDA graph; under data parallelism the gradient (with the three loss scalars
riding behind it) takes one NCCL all-reduce between the backward and the Adam kernel.

``get_models(args)`` is the reference's object (toolkit/models/__init__.py:18-46): a ``torch.nn.Module`` whose
``.model`` is the Attention net, whose ``parameters()`` are ``nn.Parameter`` views of the flat buffer under the
reference's names, and whose forward is an autograd node over the same two kernels -- so the reference's own
``train_or_eval_model`` (forward, ``cls_loss + reg_loss``, ``loss.backward()``, ``clip_grad_value_``,
``torch.optim.Adam.step()``, main-release.py:17-87) runs on it unchanged.  ``train_or_eval_model`` here is that
loop; handed this module's ``Adam`` holder instead of ``torch.optim.Adam`` it takes the fused step.
"""
from __future__ import annotations

import ctypes as C
import functools
import types

import numpy as np
import torch

from . import _lib as L

ENC = ("audio_encoder", "text_encoder", "video_encoder", "attention_mlp")


class MerFusionDims(C.Structure):
    _fields_ = [("audio_dim", C.c_int), ("text_dim", C.c_int), ("video_dim", C.c_int),
                ("hidden", C.c_int), ("out1", C.c_int), ("out2", C.c_int)]


class MerAdamHyper(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("lr", "beta1", "beta2", "eps", "weight_decay", "grad_clip")]


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


def param_shapes(audio_dim, text_dim, video_dim, hidden, out1, out2, feat_type="utt"):
    """{name: shape} of the Attention net in state_dict order: the three encoders (MLPEncoder: linear_1..3; LSTMEncoder,
    encoder.py:45-72: rnn then linear_1), attention_mlp, fc_att, fc_out_1, fc_out_2."""
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


def param_names(feat_type="utt"):
    """The Attention net's state_dict names, in order (they do not depend on the widths)."""
    return list(param_shapes(1, 1, 1, 1, 1, 1, feat_type))


def topn_param_shapes(feat_dims, hidden, out1, out2):
    """{name: shape} of Attention_TOPN in state_dict order (attention_topn.py:27-50): encoder0 .. encoder{N-1} and
    attention_mlp (MLPEncoder: linear_1..3), fc_att, fc_out_1, fc_out_2."""
    N, shapes = len(feat_dims), {}
    for i, d in enumerate(list(feat_dims) + [hidden * N]):
        e = f"encoder{i}" if i < N else "attention_mlp"
        for l, k in (("linear_1", d), ("linear_2", hidden), ("linear_3", hidden)):
            shapes[f"{e}.{l}.weight"], shapes[f"{e}.{l}.bias"] = (hidden, k), (hidden,)
    for l, o in (("fc_att", N), ("fc_out_1", out1), ("fc_out_2", out2)):
        shapes[f"{l}.weight"], shapes[f"{l}.bias"] = (o, hidden), (o,)
    return shapes


def _torch_init(shapes):
    """The initial state_dict of the reference net laid out as ``shapes``: torch's own constructors on the CPU, one per
    parameter group in dict order -- ``nn.Linear`` for each ``.weight``, ``nn.LSTM`` for each ``.rnn.weight_ih_l0``.
    When ``shapes`` follows the order in which the reference's __init__ builds its sub-modules, the values AND the
    consumption of torch's global generator are the reference's by construction."""
    sd = {}
    for name, shape in shapes.items():
        if name.endswith(".rnn.weight_ih_l0"):
            prefix, mod = name[:-len("weight_ih_l0")], torch.nn.LSTM(shape[1], shape[0] // 4, batch_first=True)
        elif name.endswith(".weight"):
            prefix, mod = name[:-len("weight")], torch.nn.Linear(shape[1], shape[0])
        else:
            continue
        sd.update((prefix + k, v) for k, v in mod.state_dict().items())
    return {k: sd[k] for k in shapes}


@functools.cache
def _api():
    """ctypes handles of the mer_fusion_* entry points, declared once, on first use; the nets bind the ones they call
    as ``_fwd``, ``_fb``, ``_step``, ``_fwd_train``, ``_bwd``, ``_fwd_frm``, ``_fb_frm`` and ``_adam``."""
    D, T = C.POINTER(MerFusionDims), C.POINTER(MerFusionTopnDims)
    vp, i32, f32, i64, u64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong, C.c_ulonglong
    return types.SimpleNamespace(
        param_count=L.declare("mer_fusion_param_count", [D], restype=i64),
        workspace_bytes=L.declare("mer_fusion_workspace_bytes", [D, i32], restype=i64),
        frm_param_count=L.declare("mer_fusion_frm_param_count", [D], restype=i64),
        frm_workspace_bytes=L.declare("mer_fusion_frm_workspace_bytes", [D, i32, i32, i32, i32], restype=i64),
        topn_param_count=L.declare("mer_fusion_topn_param_count", [T], restype=i64),
        topn_workspace_bytes=L.declare("mer_fusion_topn_workspace_bytes", [T, i32], restype=i64),
        forward=L.declare("mer_fusion_forward", [D, vp, vp, vp, vp, i32, vp, i64, vp, vp, vp, vp]),
        fwd_bwd=L.declare("mer_fusion_fwd_bwd", [D, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, u64, vp, vp, vp, i64,
                                                 vp, vp, vp, vp, vp]),
        step=L.declare("mer_fusion_step", [D, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, u64, vp, vp,
                                           C.POINTER(MerAdamHyper), vp, i64, vp, vp, vp, vp, vp]),
        forward_train=L.declare("mer_fusion_forward_train", [D, vp, vp, vp, vp, i32, f32, u64, vp, vp, vp, i64, vp,
                                                             vp, vp, vp]),
        backward=L.declare("mer_fusion_backward", [D, vp, vp, vp, vp, vp, i32, vp, vp, vp, f32, u64, vp, vp, vp, i64,
                                                   vp, vp, vp, vp]),
        frm_forward=L.declare("mer_fusion_frm_forward", [D, vp, vp, vp, vp, i32, i32, i32, i32, vp, i64, vp, vp, vp,
                                                         vp]),
        frm_fwd_bwd=L.declare("mer_fusion_frm_fwd_bwd", [D, vp, vp, vp, vp, vp, i32, i32, i32, vp, vp, i32, f32, f32,
                                                         u64, vp, vp, vp, i64, vp, vp, vp, vp, vp]),
        topn_step=L.declare("mer_fusion_topn_step", [T, vp, vp, vp, vp, vp, i32, f32, f32, u64, vp, vp, vp, i64, vp,
                                                     vp, vp, vp, vp]),
        adam=L.declare("mer_fusion_adam", [vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, f32, f32, vp, vp]))


def _size(n):
    """A parameter count or workspace size from the library; a negative one means it refused the dims or the batch."""
    n = int(n)
    if n < 0:
        L.check(2)
    return n


class _DeviceNet:
    """A device-resident fusion net: flat fp32 parameters, gradient and Adam moments in the reference's state_dict order
    (``shapes``: {name: shape}), the step counter and a workspace, with the host side every such net shares -- views by
    name, state dicts, data-parallel replicas, the Adam launch and CUDA-graph replay of a training step."""

    def __init__(self, shapes, n_params, device):
        L.check(L.lib().mer_check_device())
        self.device = torch.device(device)
        self.shapes, self.n_params = shapes, _size(n_params)
        assert sum(int(np.prod(s)) for s in shapes.values()) == self.n_params
        z = lambda: torch.zeros(self.n_params, dtype=torch.float32, device=self.device)  # noqa: E731
        self.params, self.exp_avg, self.exp_avg_sq = z(), z(), z()
        # the gradient and the three loss scalars share one allocation: ONE all-reduce under data parallelism
        self._grads_loss = torch.zeros(self.n_params + 4, dtype=torch.float32, device=self.device)
        self.grads = self._grads_loss[:self.n_params]
        self.loss = self._grads_loss[self.n_params:self.n_params + 3]
        self.step_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.training = True
        self.graph_launches = 0  # kernels launched through CUDA-graph replays (not seen by the library counter)
        self._graphs = {}
        self._adam = _api().adam

    # ---- nn.Module-flavoured surface used by the reference loop --------------------------------
    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def parameters(self):
        return [self.params]

    def named_views(self, flat=None):
        flat = self.params if flat is None else flat
        out, o = {}, 0
        for name, shape in self.shapes.items():
            k = int(np.prod(shape))
            out[name] = flat[o:o + k].view(shape)
            o += k
        return out

    def state_dict(self):
        return {k: v.clone() for k, v in self.named_views().items()}

    def load_state_dict(self, sd):
        """Accepts the reference's names with or without the ``model.`` wrapper prefix
        (toolkit/models/__init__.py wraps the net as ``.model``)."""
        for n, dst in self.named_views().items():
            src = sd[n] if n in sd else sd["model." + n]
            if isinstance(src, np.ndarray):
                src = torch.from_numpy(src)
            dst.copy_(src.to(self.device, torch.float32))
        self._graphs.clear()
        return self

    # ---- shared pieces of the steps --------------------------------------------------------------
    def _workspace(self, nbytes):
        """``self.ws``, grown to ``nbytes`` (a workspace query's answer).  Growing drops the captured graphs: they hold
        the old buffer's address."""
        nbytes = _size(nbytes)
        if self.ws.numel() < nbytes:
            self.ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self._graphs.clear()
        return self.ws

    @staticmethod
    def _mask_array(ext_masks, n):
        """ext_masks (device keep-masks; a None entry takes the counter hash) as the host ``void*[]`` the library reads
        ``n`` entries of, or None."""
        if ext_masks is None:
            return None
        ptrs = [m.data_ptr() if m is not None else None for m in ext_masks]
        return C.cast((C.c_void_p * max(n, len(ptrs)))(*ptrs), C.c_void_p)

    def _adam_update(self, world, lr, betas, eps, weight_decay, grad_clip):
        """mer_fusion_adam on ``grads`` (grad_clip 0 = off); with world > 1 the gradient and the loss terms behind it
        are summed over the ranks first."""
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(self._grads_loss)  # SUM: gradient and loss terms already carry 1 / global_batch
        L.check(self._adam(L.ptr(self.params), L.ptr(self.grads), L.ptr(self.exp_avg), L.ptr(self.exp_avg_sq),
                           self.n_params, lr, betas[0], betas[1], eps, weight_decay, 1.0, grad_clip,
                           L.ptr(self.step_counter), L.stream_ptr()))

    def _graph_step(self, key, inputs, make_outs, launch):
        """One training step through the CUDA graph cached under ``key``: ``inputs`` are copied into the graph's static
        buffers and the graph is replayed; returns its static outputs.  ``launch(*static_inputs, outs)`` enqueues the
        step on the current stream, writing into ``outs = make_outs()``.  A new key is warmed up outside capture on a
        side stream, with the state it advances restored afterwards, then captured."""
        if key not in self._graphs:
            st, outs = [x.clone() for x in inputs], make_outs()
            state = (self.params, self.exp_avg, self.exp_avg_sq, self.step_counter)
            saved = [x.clone() for x in state]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                launch(*st, outs)
            torch.cuda.current_stream().wait_stream(s)
            for dst, src in zip(state, saved):
                dst.copy_(src)
            g = torch.cuda.CUDAGraph()
            n0 = L.launch_count()
            with torch.cuda.graph(g):
                launch(*st, outs)
            self._graphs[key] = (g, (st, outs), L.launch_count() - n0)
        g, (st, outs), n_kernels = self._graphs[key]
        for dst, src in zip(st, inputs):
            dst.copy_(src, non_blocking=True)
        g.replay()
        self.graph_launches += n_kernels
        return outs

    # ---- data parallelism ----------------------------------------------------------------------
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
            raise RuntimeError(f"{type(self).__name__}: the data-parallel ranks hold different parameters "
                               "(call broadcast_from(0) after construction / load_state_dict)")
        self._replicas_checked = True


class FusionNet(_DeviceNet):
    """Device-resident Attention fusion model.  feat_type 'utt': MLP encoders on [B, D] features;
    'frm_align' / 'frm_unalign': LSTM encoders on [B, T, D] sequences (attention.py:25-33).  output_dim2 = 0 is the
    emotion-only head of the MER2024 / 25 / 26 dataloaders: vals_out is [B, 0] and the loss is CE alone.
    output_dim1 = 0 is the regression-only head of the sentiment dataloaders (CMU-MOSI / MOSEI, SIMS / SIMSv2,
    cmudata.py:20-23): emos_out is [B, 0], the loss is MSE alone and the emotion labels are never read."""

    def __init__(self, audio_dim=768, text_dim=768, video_dim=768, hidden_dim=128, output_dim1=6,
                 output_dim2=1, dropout=0.0, grad_clip=-1.0, device="cuda", max_batch=4096, seed=0,
                 feat_type="utt"):
        assert feat_type in ("utt", "frm_align", "frm_unalign"), feat_type
        self.feat_type = feat_type
        self.frm = feat_type != "utt"
        self.dims = MerFusionDims(audio_dim, text_dim, video_dim, hidden_dim, output_dim1, output_dim2)
        self.dropout, self.grad_clip, self.seed = float(dropout), float(grad_clip), int(seed)
        self.max_batch = max_batch
        api = _api()
        super().__init__(param_shapes(audio_dim, text_dim, video_dim, hidden_dim, output_dim1, output_dim2, feat_type),
                         (api.frm_param_count if self.frm else api.param_count)(C.byref(self.dims)), device)
        if not self.frm:  # one workspace for every batch up to max_batch; the frame-level one grows with the lengths
            self._workspace(api.workspace_bytes(C.byref(self.dims), max_batch))
        self._fwd, self._fb, self._step = api.forward, api.fwd_bwd, api.step
        self._fwd_train, self._bwd = api.forward_train, api.backward
        self._fwd_frm, self._fb_frm = api.frm_forward, api.frm_fwd_bwd

    def cuda(self):
        return self

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
        return self._workspace(_api().frm_workspace_bytes(C.byref(self.dims), B, a.shape[1], t.shape[1], v.shape[1]))

    def _launch_step(self, a, t, v, emo, val, outs, lr, betas, eps, wd, world, ext_masks, global_batch=None,
                     fused_adam=True):
        B = a.shape[0]
        inv = 1.0 / (global_batch if global_batch is not None else B * world)
        masks = self._mask_array(ext_masks, 4)
        clip = self.grad_clip if self.grad_clip != -1 else 0.0
        seed = _dist_seed(self.seed, world)
        feats, emos_out, vals_out = outs
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
        self._adam_update(world, lr, betas, eps, wd, clip)

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
            outs = self._bufs(B)
            self._launch_step(a.contiguous(), t.contiguous(), v.contiguous(), emo.contiguous(), val.contiguous(), outs,
                              lr, betas, eps, weight_decay, world_size, ext_masks, global_batch, fused_adam)
            return self.loss, outs[1], outs[2]
        if self.frm:
            self._frm_ws(B, a, t, v)  # sized (and graphs invalidated on growth) before any capture
        key = (B, tuple(a.shape[1:]), tuple(t.shape[1:]), tuple(v.shape[1:]), lr, betas, eps, weight_decay,
               world_size, self.dropout, self.grad_clip)
        _, emos_out, vals_out = self._graph_step(
            key, (a, t, v, emo, val), lambda: self._bufs(B),
            lambda *x: self._launch_step(*x, lr, betas, eps, weight_decay, world_size, None))
        return self.loss, emos_out, vals_out

    # ---- the two halves of the autograd node (utterance-level net) -----------------------------------
    def forward_train(self, a, t, v, ext_masks=None):
        """Train-mode forward (dropout from (seed, step_counter) or ext_masks) -> (features, emos_out, vals_out)."""
        assert not self.frm, "the autograd node covers the utterance-level Attention net"
        B = a.shape[0]
        assert B <= self.max_batch
        feats, emos, vals = self._bufs(B)
        L.check(self._fwd_train(C.byref(self.dims), L.ptr(self.params), L.ptr(a), L.ptr(t), L.ptr(v), B,
                                self.dropout, self.seed, L.ptr(self.step_counter), self._mask_array(ext_masks, 4),
                                L.ptr(self.ws), self.ws.numel(), L.ptr(feats), L.ptr(emos), L.ptr(vals),
                                L.stream_ptr()))
        return feats, emos, vals

    def backward(self, a, t, v, d_feats, d_emos, d_vals, ext_masks=None):
        """d(loss)/d(params) into ``self.grads`` from the upstream gradients of forward_train's outputs (None =
        zero); must see the same inputs, masks and step counter as the forward it differentiates."""
        B = a.shape[0]
        feats, emos, vals = self._bufs(B)
        c = lambda g: None if g is None else g.contiguous().float()  # noqa: E731
        d_feats, d_emos, d_vals = c(d_feats), c(d_emos), c(d_vals)
        L.check(self._bwd(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(a), L.ptr(t),
                          L.ptr(v), B, L.ptr(d_feats), L.ptr(d_emos), L.ptr(d_vals), self.dropout, self.seed,
                          L.ptr(self.step_counter), self._mask_array(ext_masks, 4), L.ptr(self.ws),
                          self.ws.numel(), L.ptr(feats), L.ptr(emos), L.ptr(vals), L.stream_ptr()))
        return self.grads


class MerFusionTopnDims(C.Structure):
    _fields_ = [("n_feats", C.c_int), ("feat_dims", C.c_int * 18), ("hidden", C.c_int), ("out1", C.c_int),
                ("out2", C.c_int)]


class TopnFusionNet(_DeviceNet):
    """Attention_TOPN (MER2026_Track1/toolkit/models/attention_topn.py): the utterance-level fusion net over
    N <= 18 features ``batch['feat0'] .. batch['feat{N-1}']`` ([B, feat_dims[i]] each).  output_dim2 may be 0."""

    def __init__(self, feat_dims, hidden_dim=128, output_dim1=6, output_dim2=1, dropout=0.0, grad_clip=-1.0,
                 device="cuda", seed=0):
        assert 1 <= len(feat_dims) <= 18
        self.feat_dims = [int(d) for d in feat_dims]
        self.dims = MerFusionTopnDims(len(feat_dims), (C.c_int * 18)(*self.feat_dims), hidden_dim, output_dim1,
                                      output_dim2)
        self.dropout, self.grad_clip, self.seed = float(dropout), float(grad_clip), int(seed)
        super().__init__(topn_param_shapes(self.feat_dims, hidden_dim, output_dim1, output_dim2),
                         _api().topn_param_count(C.byref(self.dims)), device)
        self._step = _api().topn_step

    def _run(self, feats, emo, val, ext_masks, world, global_batch=None):
        B = feats[0].shape[0]
        ws = self._workspace(_api().topn_workspace_bytes(C.byref(self.dims), B))
        feats = [f.contiguous() for f in feats]
        fp = (C.c_void_p * len(feats))(*[f.data_ptr() for f in feats])
        d = self.dims
        out = [torch.empty(B, n, dtype=torch.float32, device=self.device) for n in (d.hidden, d.out1, d.out2)]
        L.check(self._step(C.byref(d), L.ptr(self.params), L.ptr(self.grads), C.cast(fp, C.c_void_p),
                           L.ptr(emo), L.ptr(val), B,
                           1.0 / (global_batch if global_batch is not None else B * world),
                           self.dropout if emo is not None else 0.0, _dist_seed(self.seed, world),
                           L.ptr(self.step_counter), self._mask_array(ext_masks, d.n_feats + 1),
                           L.ptr(ws), ws.numel(), L.ptr(self.loss), L.ptr(out[0]), L.ptr(out[1]),
                           L.ptr(out[2]), L.stream_ptr()))
        return out

    def forward(self, batch):
        """batch: {'feat0': [B, d0], ...}; eval-mode forward -> (features, emos_out, vals_out, interloss)."""
        feats = [batch[f"feat{i}"] for i in range(len(self.feat_dims))]
        f, e, v = self._run(feats, None, None, None, 1)
        return f, e, v, torch.zeros((), dtype=torch.int64, device=self.device)

    __call__ = forward

    def train_step(self, feats, emo, val, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, world_size=1,
                   ext_masks=None, global_batch=None):
        """One optimisation step (forward, CE + MSE, backward, optional all-reduce, Adam).  world_size > 1: this rank's
        slice of a data-parallel batch of ``global_batch`` rows (default: batch * world_size); the gradient and the
        loss returned are the global ones."""
        assert emo.dtype == torch.int64 and val.dtype == torch.float32
        if world_size > 1:
            self.check_replicas(world_size)
        _, eo, vo = self._run(feats, emo.contiguous(), val.contiguous(), ext_masks, world_size, global_batch)
        self._adam_update(world_size, lr, betas, eps, weight_decay, self.grad_clip if self.grad_clip != -1 else 0.0)
        return self.loss, eo, vo


def reference_init(feat_type, audio_dim, text_dim, video_dim, hidden, out1, out2):
    """The state_dict ``get_models(args)`` of the reference starts from: torch's own ``nn.Linear`` / ``nn.LSTM``
    constructors, called on the CPU in the order Attention.__init__ builds its sub-modules (attention.py:25-40;
    MLPEncoder: linear_1..3, encoder.py:25-27; LSTMEncoder: rnn then linear_1, encoder.py:59-61), so the values AND
    the consumption of torch's global generator are the reference's by construction."""
    return _torch_init(param_shapes(audio_dim, text_dim, video_dim, hidden, out1, out2, feat_type))


def reference_init_topn(feat_dims, hidden, out1, out2):
    """reference_init for Attention_TOPN: torch's own nn.Linear constructors on the CPU in the order
    Attention_TOPN.__init__ builds them (attention_topn.py:27-50): encoder0 .. encoder{N-1} (MLPEncoder: linear_1..3),
    attention_mlp, fc_att, fc_out_1, fc_out_2 -- nn.Linear(hidden, 0) when out2 == 0, an empty weight and bias."""
    return _torch_init(topn_param_shapes(feat_dims, hidden, out1, out2))


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
                                device=getattr(args, "device", "cuda"), seed=getattr(args, "seed", 0))
            # the reference's initial weights, drawn here and not in TopnFusionNet.__init__: callers that construct
            # the net directly and load their own state dict draw nothing from torch's generator
            net.load_state_dict(reference_init_topn(args.audio_dim, args.hidden_dim, args.output_dim1,
                                                    args.output_dim2))
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


def mer2026_calculate_results(emo_probs=(), emo_labels=(), val_preds=(), val_labels=()):
    """MER2026_Track1/toolkit/dataloader/mer2026.py:132-145 (MER2024 / MER2025 have the same rule): emotion metrics
    only, the valence arguments are ignored."""
    from sklearn.metrics import accuracy_score, f1_score
    emo_preds = np.argmax(emo_probs, 1)
    acc = accuracy_score(emo_labels, emo_preds)
    f1 = f1_score(emo_labels, emo_preds, average="weighted")
    return dict(emoprobs=emo_probs, emolabels=emo_labels, emoacc=acc, emofscore=f1), f"f1:{f1:.4f}_acc:{acc:.4f}"


def sentiment_calculate_results(emo_probs=(), emo_labels=(), val_preds=(), val_labels=()):
    """cmudata.py:69-84 (sims.py, simsv2.py and crossdim.py have the same rule): acc-2 and weighted F1 of the sign of
    the valence over the clips whose label is not 0; the emotion arguments are ignored."""
    from sklearn.metrics import accuracy_score, f1_score
    labels, preds = np.asarray(val_labels).reshape(-1), np.asarray(val_preds).reshape(-1)
    keep = labels != 0
    acc = accuracy_score(labels[keep] > 0, preds[keep] > 0)
    f1 = f1_score(labels[keep] > 0, preds[keep] > 0, average="weighted")
    return dict(valpreds=val_preds, vallabels=val_labels, emoacc=acc, emofscore=f1), f"f1:{f1:.4f}_acc:{acc:.4f}"


def train_or_eval_model(args, model, reg_loss, cls_loss, dataloader, epoch, optimizer=None, train=False,
                        calculate_results=None, world_size=1):
    """main-release.py:17-87: same arguments, same ``save_results`` dict (names, loss, then the keys of
    ``dataloader_class.calculate_results``; default: the MER2023 rule).  The CE loss and the emotion scores enter only
    when ``args.output_dim1 != 0``, the regression loss and the valence predictions only when ``args.output_dim2 != 0``
    (main-release.py:51-58); pass ``mer2026_calculate_results`` for the MER2024 / 25 / 26 corpora and
    ``sentiment_calculate_results`` for the sentiment corpora.  With a ``torch.optim`` optimizer this IS the
    reference loop (zero_grad, forward, ``cls_loss + reg_loss``, backward, clip_grad_value_, step) running on the
    autograd node; with this module's ``Adam`` holder each training batch is one fused FusionNet.train_step."""
    vidnames, val_preds, val_labels, emo_probs, emo_labels, losses = [], [], [], [], [], []
    assert not train or optimizer is not None
    has_emo = getattr(args, "output_dim1", 6) != 0
    has_val = getattr(args, "output_dim2", 1) != 0
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
            kw = dict(lr=optimizer.lr, betas=optimizer.betas, eps=optimizer.eps, weight_decay=optimizer.weight_decay,
                      world_size=world_size)
            if isinstance(net, TopnFusionNet):
                feats = [batch[f"feat{i}"] for i in range(len(net.feat_dims))]
                loss3, emos_out, vals_out = net.train_step(feats, emos.long(), vals.float().view(-1, 1), **kw)
            else:
                loss3, emos_out, vals_out = net.train_step(
                    batch["audios"], batch["texts"], batch["videos"], emos.long(), vals.float().view(-1, 1), **kw)
            loss = loss3[2]
        else:
            _, emos_out, vals_out, interloss = model(batch)
            loss = interloss
            if has_emo:
                loss = loss + cls_loss(emos_out, emos)
            if has_val:
                loss = loss + reg_loss(vals_out, vals)
        if has_emo:
            emo_probs.append(emos_out.data.cpu().numpy())
            emo_labels.append(emos.data.cpu().numpy())
        if has_val:
            val_preds.append(vals_out.data.cpu().numpy())
            val_labels.append(vals.data.cpu().numpy())
        losses.append(loss.data.cpu().numpy())
        if train and not fused:
            loss.backward()
            clip = getattr(getattr(model, "model", model), "grad_clip", -1)
            if clip != -1:
                torch.nn.utils.clip_grad_value_([p for p in model.parameters() if p.requires_grad], clip)
            optimizer.step()
    if has_emo:
        emo_probs, emo_labels = np.concatenate(emo_probs), np.concatenate(emo_labels)
    if has_val:
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
