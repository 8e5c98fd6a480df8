"""The MER2023 challenge baseline nets on the device -- ``MLP`` and ``Attention`` of MER2023/main-release.py:226-290
with a free ``--layers`` list -- and their training step (CELoss + MSELoss, torch.optim.Adam with coupled L2,
:293-369), driving csrc/fusion_mlp.cu through libmer_b200.so.

``MlpFusionNet`` owns flat fp32 parameter / gradient / Adam-moment buffers in the reference's state_dict order.  Its
``train_step`` is one row-parallel cluster kernel (forward, losses, data gradients), one weight-gradient kernel and
mer_fusion_adam, replayed as a CUDA graph; ``forward`` is the eval-mode pass.  The reference builds both nets without
their ``dropout`` argument (:601-612), so dropout is 0.3 whatever ``--dropout`` says; that is the default here.
"""
from __future__ import annotations

import ctypes as C
import functools
import types

import torch

from . import _lib as L
from .fusion import MerAdamHyper, _DeviceNet, _torch_init

KINDS = {"mlp": 0, "attention": 1}
CHAINS = {"mlp": ("module",), "attention": ("audio_mlp", "text_mlp", "video_mlp", "attention_mlp")}
MAX_LAYERS = 8
REFERENCE_DROPOUT = 0.3   # MLP / Attention default, the value the reference trains with (main-release.py:227, :249)


class MerMlpDims(C.Structure):
    _fields_ = [("kind", C.c_int), ("audio_dim", C.c_int), ("text_dim", C.c_int), ("video_dim", C.c_int),
                ("n_layers", C.c_int), ("layers", C.c_int * MAX_LAYERS), ("out1", C.c_int), ("out2", C.c_int)]


def parse_layers(layers):
    """``--layers`` '256,128' -> [256, 128] (the reference's ``list(map(int, layers.split(',')))``)."""
    return [int(x) for x in layers.split(",")] if isinstance(layers, str) else [int(x) for x in layers]


def param_shapes(kind, audio_dim, text_dim, video_dim, layers, out1=6, out2=1):
    """{name: shape} in state_dict order: ``module.{0,3,..}.weight/.bias``, fc_out_1, fc_out_2 for the MLP;
    audio_mlp, text_mlp, video_mlp, attention_mlp (each ``{0,3,..}``), fc_att, fc_out_1, fc_out_2 for Attention.
    The Sequential's indices step by 3: each layer is Linear, ReLU, Dropout."""
    layers = parse_layers(layers)
    ins = {"module": audio_dim + text_dim + video_dim, "audio_mlp": audio_dim, "text_mlp": text_dim,
           "video_mlp": video_dim, "attention_mlp": 3 * layers[-1]}
    shapes = {}
    for ch in CHAINS[kind]:
        k = ins[ch]
        for i, n in enumerate(layers):
            shapes[f"{ch}.{3 * i}.weight"], shapes[f"{ch}.{3 * i}.bias"] = (n, k), (n,)
            k = n
    heads = ([("fc_att", 3)] if kind == "attention" else []) + [("fc_out_1", out1), ("fc_out_2", out2)]
    for name, o in heads:
        shapes[f"{name}.weight"], shapes[f"{name}.bias"] = (o, layers[-1]), (o,)
    return shapes


def reference_init(kind, audio_dim, text_dim, video_dim, layers, out1=6, out2=1):
    """The state_dict ``MLP(...)`` / ``Attention(...)`` of main-release.py:601-612 starts from: torch's own
    ``nn.Linear`` constructors on the CPU, in the order the reference's __init__ calls them (ReLU and Dropout draw
    nothing), so the values and the consumption of torch's global generator are the reference's by construction."""
    return _torch_init(param_shapes(kind, audio_dim, text_dim, video_dim, layers, out1, out2))


def mask_shapes(kind, layers, batch):
    """The [batch, width] keep-masks of one training forward, in the reference's call order: every layer of each chain,
    chains in forward order (audio, text, video, attention for the Attention net)."""
    return [(batch, n) for _ in CHAINS[kind] for n in parse_layers(layers)]


def check_batch(kind, batch):
    """The Attention net refuses a one-row batch: the reference squeezes its [1, L] fused features to a vector
    (main-release.py:287), and the CE loss or the concatenation of the outputs that follows fails."""
    if kind == "attention" and batch < 2:
        raise ValueError("the MER2023 Attention net needs at least 2 rows per batch: the reference squeezes a 1-row "
                         "batch's fused features to a vector and fails (main-release.py:287); use a batch size that "
                         "leaves no batch of one row")


@functools.cache
def _api():
    """ctypes handles of the mer_mlp_* entry points, declared once, on first use (bound as ``_fwd`` and ``_step``)."""
    D = C.POINTER(MerMlpDims)
    vp, i32, f32, i64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong
    return types.SimpleNamespace(
        param_count=L.declare("mer_mlp_param_count", [D], restype=i64),
        workspace_bytes=L.declare("mer_mlp_workspace_bytes", [D, i32], restype=i64),
        forward=L.declare("mer_mlp_forward", [D, vp, vp, vp, vp, i32, vp, i64, vp, vp, vp, vp]),
        train_step=L.declare("mer_mlp_train_step", [D, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, C.c_ulonglong,
                                                    vp, vp, C.POINTER(MerAdamHyper), vp, i64, vp, vp, vp, vp, vp]))


class MlpFusionNet(_DeviceNet):
    """Device-resident MLP / Attention net of MER2023/main-release.py.  kind: 'mlp' | 'attention'; layers: the
    ``--layers`` string or list."""

    def __init__(self, kind, audio_dim, text_dim, video_dim, layers="256,128", output_dim1=6, output_dim2=1,
                 dropout=REFERENCE_DROPOUT, device="cuda", max_batch=1024, seed=0):
        assert kind in KINDS, kind
        self.kind, self.layers = kind, parse_layers(layers)
        assert 1 <= len(self.layers) <= MAX_LAYERS, f"--layers takes 1..{MAX_LAYERS} entries, got {self.layers}"
        self.dropout, self.seed, self.max_batch = float(dropout), int(seed), int(max_batch)
        lay = (C.c_int * MAX_LAYERS)(*(self.layers + [0] * (MAX_LAYERS - len(self.layers))))
        self.dims = MerMlpDims(KINDS[kind], audio_dim, text_dim, video_dim, len(self.layers), lay, output_dim1,
                               output_dim2)
        api = _api()
        super().__init__(param_shapes(kind, audio_dim, text_dim, video_dim, self.layers, output_dim1, output_dim2),
                         api.param_count(C.byref(self.dims)), device)
        self._workspace(api.workspace_bytes(C.byref(self.dims), max(self.max_batch, 2)))
        self._fwd, self._step = api.forward, api.train_step

    # ---- forward / step --------------------------------------------------------------------------
    def _outs(self, B):
        f = lambda n: torch.empty(B, n, dtype=torch.float32, device=self.device)  # noqa: E731
        return f(self.layers[-1]), f(self.dims.out1), f(self.dims.out2)

    def _check(self, B):
        check_batch(self.kind, B)
        if B > self.max_batch:
            raise ValueError(f"batch of {B} rows, the net was built for at most {self.max_batch}")

    def forward(self, a, t, v):
        """Eval-mode forward of [B, D] fp32 device features -> (features, emos_out, vals_out)."""
        B = a.shape[0]
        self._check(B)
        a, t, v = a.contiguous(), t.contiguous(), v.contiguous()
        feats, emos, vals = self._outs(B)
        L.check(self._fwd(C.byref(self.dims), L.ptr(self.params), L.ptr(a), L.ptr(t), L.ptr(v), B,
                          L.ptr(self.ws), self.ws.numel(), L.ptr(feats), L.ptr(emos), L.ptr(vals),
                          L.stream_ptr()))
        return feats, emos, vals

    __call__ = forward

    def _launch(self, a, t, v, emo, val, outs, lr, betas, eps, weight_decay, ext_masks, update):
        B = a.shape[0]
        masks = self._mask_array(ext_masks, len(CHAINS[self.kind]) * len(self.layers))
        hyper = MerAdamHyper(lr, betas[0], betas[1], eps, weight_decay, 0.0)
        L.check(self._step(C.byref(self.dims), L.ptr(self.params), L.ptr(self.grads), L.ptr(self.exp_avg),
                           L.ptr(self.exp_avg_sq), L.ptr(a), L.ptr(t), L.ptr(v), L.ptr(emo), L.ptr(val), B,
                           self.dropout, self.seed, L.ptr(self.step_counter), masks,
                           C.byref(hyper) if update else None, L.ptr(self.ws), self.ws.numel(),
                           L.ptr(self.loss), L.ptr(outs[0]), L.ptr(outs[1]), L.ptr(outs[2]), L.stream_ptr()))

    def train_step(self, a, t, v, emo, val, lr=1e-4, weight_decay=1e-5, betas=(0.9, 0.999), eps=1e-8,
                   ext_masks=None, use_graph=True, update=True):
        """One step of main-release.py:334-369 on a device batch: train-mode forward, CE + MSE, backward, Adam.
        Returns (loss[3] = {CE, MSE, total}, features, emos_out, vals_out), the train-mode outputs the reference's
        train F1 is computed from.  ext_masks: None (counter-hash masks) or the keep-masks of mask_shapes.
        update=False leaves the parameters, the Adam moments and the step counter alone (gradient in ``grads``)."""
        B = a.shape[0]
        self._check(B)
        assert emo.dtype == torch.int64 and val.dtype == torch.float32
        val = val.reshape(B, -1)
        if not use_graph or ext_masks is not None or not update:
            outs = self._outs(B)
            self._launch(a.contiguous(), t.contiguous(), v.contiguous(), emo.contiguous(), val.contiguous(), outs,
                         lr, betas, eps, weight_decay, ext_masks, update)
            return (self.loss, *outs)
        outs = self._graph_step((B, lr, betas, eps, weight_decay), (a, t, v, emo, val), lambda: self._outs(B),
                                lambda *x: self._launch(*x, lr, betas, eps, weight_decay, None, True))
        return (self.loss, *outs)
