"""ORACLE (test infrastructure -- never imported by the product path).

CPU restatement (torch autograd, fp32) of the MER2023 challenge baseline nets and their training step:
  MER2023/main-release.py:226-245 (MLP: Linear -> ReLU -> Dropout per --layers entry over A | T | V, two heads),
  :248-290 (Attention: such a chain per modality, attention_mlp over their concat, fc_att, weighted sum, two heads),
  :293-315 (CELoss, MSELoss), :363-369 and :618 (loss = CE + MSE, backward, Adam(lr, weight_decay=l2)).
Dropout keep-masks are explicit inputs, one per Dropout call in the reference's forward order, applied as torch's CPU
dropout applies them (x * (keep / (1 - p))).  Pinned against the reference itself by
tests/golden/make_golden_mer2023_baseline.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

CHAINS = {"mlp": ("module",), "attention": ("audio_mlp", "text_mlp", "video_mlp", "attention_mlp")}


def _chain(sd, prefix, x, n_layers, masks, p):
    for i in range(n_layers):
        x = F.relu(F.linear(x, sd[f"{prefix}.{3 * i}.weight"], sd[f"{prefix}.{3 * i}.bias"]))
        if masks is not None:
            x = x * masks.pop(0).to(x.dtype).div_(1 - p)
    return x


def forward(sd, kind, a, t, v, masks=None, p=0.3):
    """MLP.forward / Attention.forward -> (features, emos_out, vals_out).  masks: None (eval) or the keep-masks of every
    Dropout call in forward order.  A one-row Attention batch is refused (the reference's squeeze() breaks on it)."""
    n_layers = sum(1 for k in sd if k.startswith(CHAINS[kind][0] + ".") and k.endswith(".weight"))
    m = None if masks is None else list(masks)
    if kind == "mlp":
        feats = _chain(sd, "module", torch.cat([a, t, v], dim=1), n_layers, m, p)
    else:
        if a.shape[0] < 2:
            raise ValueError("the Attention net needs at least 2 rows per batch")
        hs = [_chain(sd, ch, x, n_layers, m, p) for ch, x in zip(CHAINS[kind][:3], (a, t, v))]
        att = F.linear(_chain(sd, "attention_mlp", torch.cat(hs, dim=1), n_layers, m, p), sd["fc_att.weight"],
                       sd["fc_att.bias"])
        # squeeze(2): the reference's squeeze() would also drop a last layer of width 1 (and then fail in fc_out_1)
        feats = torch.matmul(torch.stack(hs, dim=2), att.unsqueeze(2)).squeeze(2)
    return feats, F.linear(feats, sd["fc_out_1.weight"], sd["fc_out_1.bias"]), \
        F.linear(feats, sd["fc_out_2.weight"], sd["fc_out_2.bias"])


def losses(emos_out, vals_out, emos, vals):
    """CELoss + MSELoss (main-release.py:293-315).  The targets are flattened rather than squeezed: the same for two or
    more rows, and defined for one (the reference's squeeze() leaves a 0-d target there, which nll_loss rejects)."""
    ce = F.nll_loss(F.log_softmax(emos_out, 1), emos.reshape(-1).long(), reduction="sum") / len(emos_out)
    mse = F.mse_loss(vals_out.view(-1, 1), vals.view(-1, 1), reduction="sum") / len(vals_out)
    return ce, mse


class Net:
    """One fold's model and optimiser, with the step / eval surface of mertools_b200.fusion_mlp.MlpFusionNet, so the
    MER2023 trainer's host loop can run on it unchanged."""

    def __init__(self, kind, state_dict, dropout=0.3):
        self.kind, self.p = kind, dropout
        self.sd = {k: torch.tensor(np.asarray(v), dtype=torch.float32, requires_grad=True)
                   for k, v in state_dict.items()}
        self.opt = None

    def state_dict(self):
        return {k: v.detach().clone() for k, v in self.sd.items()}

    def forward(self, a, t, v):
        with torch.no_grad():
            return forward(self.sd, self.kind, a, t, v)

    __call__ = forward

    def train_step(self, a, t, v, emo, val, lr=1e-4, weight_decay=1e-5, ext_masks=None, **_):
        if self.opt is None:
            self.opt = torch.optim.Adam(list(self.sd.values()), lr=lr, weight_decay=weight_decay)
        assert ext_masks is not None, "the oracle takes its dropout masks as inputs"
        self.opt.zero_grad()
        feats, eo, vo = forward(self.sd, self.kind, a, t, v, ext_masks, self.p)
        ce, mse = losses(eo, vo, emo, val.float())
        loss = ce + mse
        loss.backward()
        self.opt.step()
        return torch.stack([ce, mse, loss]).detach(), feats.detach(), eo.detach(), vo.detach()
