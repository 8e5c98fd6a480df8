"""ORACLE (test infrastructure — never imported by the product path).

CPU restatement (torch autograd, fp32) of the Attention fusion net, its losses and the training
step of the reference:
  MERBench/toolkit/models/attention.py:8-57, toolkit/models/modules/encoder.py:9-41 (MLPEncoder),
  toolkit/utils/loss.py:5-28, main-release.py:31-66 (zero_grad, forward, loss = interloss + CE + MSE,
  backward, optional clip_grad_value_, Adam(lr, weight_decay=l2) :205).
Dropout masks are explicit inputs (the reference's nn.Dropout draws them from the global CPU
generator; a CUDA run cannot reproduce that stream, SURVEY.md §7) so both sides use the same masks.
Pinned against the reference's own classes by tests/golden/make_golden.py (fusion_golden.npz).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

ENC = ("audio_encoder", "text_encoder", "video_encoder", "attention_mlp")


def _mlp(sd, prefix, x, mask, p):
    """MLPEncoder.forward (encoder.py:30-41): dropout -> 3 x (Linear + ReLU)."""
    if mask is not None:
        x = x * mask / (1.0 - p)
    for l in ("linear_1", "linear_2", "linear_3"):
        x = F.relu(F.linear(x, sd[f"{prefix}.{l}.weight"], sd[f"{prefix}.{l}.bias"]))
    return x


def _lstm_encoder(sd, prefix, x, mask, p):
    """LSTMEncoder.forward (encoder.py:62-72): one-layer nn.LSTM over [B, T, D] (zero state, gate order
    i, f, g, o), final hidden state -> dropout -> linear_1 (no activation)."""
    w_ih, w_hh = sd[f"{prefix}.rnn.weight_ih_l0"], sd[f"{prefix}.rnn.weight_hh_l0"]
    b_ih, b_hh = sd[f"{prefix}.rnn.bias_ih_l0"], sd[f"{prefix}.rnn.bias_hh_l0"]
    B, T, _ = x.shape
    H = w_hh.shape[1]
    h = torch.zeros(B, H, dtype=x.dtype, device=x.device)
    c = torch.zeros(B, H, dtype=x.dtype, device=x.device)
    for t in range(T):
        g = F.linear(x[:, t], w_ih, b_ih) + F.linear(h, w_hh, b_hh)
        i, f, gg, o = g.chunk(4, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
    if mask is not None:
        h = h * mask / (1.0 - p)
    return F.linear(h, sd[f"{prefix}.linear_1.weight"], sd[f"{prefix}.linear_1.bias"])


def attention_forward(sd, audios, texts, videos, masks=None, p=0.0):
    """Attention.forward (attention.py:36-57).  masks: None (eval) or 4 keep-masks
    [audio, text, video, concat].  Returns (features, emos_out, vals_out).  Frame-level checkpoints
    (feat_type frm_align / frm_unalign, attention.py:29-33: LSTMEncoder per modality, inputs [B, T, D], masks
    0..2 on the [B, H] final hidden states) are recognised by their rnn.* parameters."""
    m = masks or (None, None, None, None)
    enc = _lstm_encoder if "audio_encoder.rnn.weight_ih_l0" in sd else _mlp
    ha = enc(sd, "audio_encoder", audios, m[0], p)
    ht = enc(sd, "text_encoder", texts, m[1], p)
    hv = enc(sd, "video_encoder", videos, m[2], p)
    cat = torch.cat([ha, ht, hv], dim=1)
    att = F.linear(_mlp(sd, "attention_mlp", cat, m[3], p), sd["fc_att.weight"], sd["fc_att.bias"])
    fused = torch.matmul(torch.stack([ha, ht, hv], dim=2), att.unsqueeze(2)).squeeze(2)
    emos = F.linear(fused, sd["fc_out_1.weight"], sd["fc_out_1.bias"])
    vals = F.linear(fused, sd["fc_out_2.weight"], sd["fc_out_2.bias"])
    return fused, emos, vals


def attention_topn_forward(sd, feats, masks=None, p=0.0):
    """Attention_TOPN.forward (MER2026_Track1/toolkit/models/attention_topn.py:55-90): one MLPEncoder per
    feature (encoder0..), attention_mlp on the concat, fc_att -> one weight per feature (no softmax), weighted
    sum.  masks: None or len(feats) + 1 keep-masks (inputs, then the concat)."""
    n = len(feats)
    m = masks or [None] * (n + 1)
    hs = [_mlp(sd, f"encoder{i}", feats[i], m[i], p) for i in range(n)]
    att = F.linear(_mlp(sd, "attention_mlp", torch.cat(hs, dim=1), m[n], p), sd["fc_att.weight"], sd["fc_att.bias"])
    fused = torch.matmul(torch.stack(hs, dim=2), att.unsqueeze(2)).squeeze(2)
    return fused, F.linear(fused, sd["fc_out_1.weight"], sd["fc_out_1.bias"]), \
        F.linear(fused, sd["fc_out_2.weight"], sd["fc_out_2.bias"])


def losses(emos_out, vals_out, emos, vals):
    """CELoss + MSELoss (loss.py:11-28)."""
    ce = F.nll_loss(F.log_softmax(emos_out, 1), emos.long(), reduction="sum") / len(emos_out)
    mse = F.mse_loss(vals_out.view(-1, 1), vals.view(-1, 1), reduction="sum") / len(vals_out)
    return ce, mse


class Trainer:
    """State of one reference training run: parameters as leaf tensors + torch.optim.Adam."""

    def __init__(self, state_dict, lr=1e-3, l2=1e-5, grad_clip=-1.0, dropout=0.0):
        self.sd = {k: torch.tensor(np.asarray(v), dtype=torch.float32, requires_grad=True)
                   for k, v in state_dict.items()}
        self.opt = torch.optim.Adam(list(self.sd.values()), lr=lr, weight_decay=l2)
        self.grad_clip, self.p = grad_clip, dropout

    def step(self, a, t, v, emos, vals, masks=None):
        """main-release.py:31-66 for one batch.  Returns (ce, mse, total, emos_out, vals_out, grads)."""
        self.opt.zero_grad()
        if "encoder0.linear_1.weight" in self.sd:  # Attention_TOPN: `a` is the list of features
            _, eo, vo = attention_topn_forward(self.sd, a, masks, self.p)
        else:
            _, eo, vo = attention_forward(self.sd, a, t, v, masks, self.p)
        ce, mse = losses(eo, vo, emos, vals)
        loss = ce + mse
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in self.sd.items()}
        if self.grad_clip != -1:
            torch.nn.utils.clip_grad_value_(list(self.sd.values()), self.grad_clip)
        self.opt.step()
        return float(ce.detach()), float(mse.detach()), float(loss.detach()), eo.detach(), vo.detach(), grads
