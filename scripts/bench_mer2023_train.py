"""Wall time of MER2023 baseline training runs (mertools_b200.main_release_mer2023): 5 folds x 100 epochs of
``--model_type mlp`` and ``--model_type attention`` with the default ``--layers 256,128``, batch 32, l2 1e-5, in two
settings: the trainer's defaults (lr 1e-4, --test_sets test1,test2) and MER2023/run_release.sh's (lr 1e-3,
--test_sets test3).  The corpus is synthetic at the real MER2023 sizes (3,373 train / 411 test1 / 412 test2 / 834 test3
clips: the label-6way.npz of the MER2023 release, SURVEY.md row 27) with 1024-wide A / T / V features (the width of
chinese-hubert-large, chinese-macbert-large and MANet).

Each epoch is what the CLI runs (main_release_mer2023.run_pass): a training pass over the fold's train part in
SubsetRandomSampler order, an eval pass over its eval part and a pass over each test set, every pass ending in the
reference's F1 / MSE on the host.  Two arms on the same GPU, same data, same loaders:
  ours   MlpFusionNet: one CUDA-graph replay per training batch (row kernel, weight-gradient kernel, Adam), eval
         forwards on the device;
  eager  the repository's torch restatement of the nets (oracle/mer2023.py) on the GPU, fp32, dropout masks drawn with
         torch.rand, with torch.optim.Adam -- the reference's own loop run in torch eager.
Prints one JSON line per (arm, model, setting) and the card name and power limit beside the numbers; --out also writes
them to a file.  --folds / --epochs shorten a run (the eager arm is slow: say so beside its numbers).
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"train": 3373, "test1": 411, "test2": 412, "test3": 834}
WIDTH = 1024
SETTINGS = {"default": (1e-4, ("test1", "test2")), "run_release": (1e-3, ("test3",))}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def split(n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    s = types.SimpleNamespace(names=[f"c{seed}_{i}" for i in range(n)])
    s.a, s.t, s.v = (torch.randn(n, WIDTH, generator=g).to(dev) for _ in range(3))
    s.emo = torch.randint(0, 6, (n,), generator=g).to(dev)
    s.val = (torch.rand(n, generator=g) * 6 - 3).to(dev)
    return s


class EagerNet:
    """oracle/mer2023.py's forward on the GPU with torch.optim.Adam and torch.rand keep-masks."""

    def __init__(self, kind, sd, layers, dev, lr, l2):
        from oracle import mer2023 as O
        self.O, self.kind, self.layers = O, kind, layers
        self.sd = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
        self.opt = torch.optim.Adam(list(self.sd.values()), lr=lr, weight_decay=l2)

    def __call__(self, a, t, v):
        with torch.no_grad():
            return self.O.forward(self.sd, self.kind, a, t, v)

    def train_step(self, a, t, v, emo, val, **_):
        from mertools_b200.fusion_mlp import mask_shapes
        masks = [torch.rand(s, device=a.device) >= 0.3 for s in mask_shapes(self.kind, self.layers, a.shape[0])]
        self.opt.zero_grad()
        f, eo, vo = self.O.forward(self.sd, self.kind, a, t, v, masks, 0.3)
        ce, mse = self.O.losses(eo, vo, emo, val)
        (ce + mse).backward()
        self.opt.step()
        return torch.stack([ce, mse, ce + mse]).detach(), f.detach(), eo.detach(), vo.detach()


def run(arm, kind, setting, folds, epochs, dev):
    from mertools_b200 import main_release as MR
    from mertools_b200 import main_release_mer2023 as M
    from mertools_b200.fusion_mlp import MlpFusionNet, reference_init
    lr, test_sets = SETTINGS[setting]
    layers = "256,128"
    train = split(SIZES["train"], 1, dev)
    tests = [split(SIZES[ts], 2 + i, dev) for i, ts in enumerate(test_sets)]
    random.seed(0)
    torch.manual_seed(0)
    fold_idx = MR.random_split_indexes(SIZES["train"], 5)[:folds]
    trl, evl, tel = MR.get_loaders(SIZES["train"], fold_idx, [SIZES[ts] for ts in test_sets], 32)
    args = types.SimpleNamespace(model_type=kind, savewhole=False)
    steps = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(folds):
        sd = reference_init(kind, WIDTH, WIDTH, WIDTH, layers)
        if arm == "ours":
            net = MlpFusionNet(kind, WIDTH, WIDTH, WIDTH, layers, device=dev, max_batch=32, seed=f).load_state_dict(sd)
        else:
            net = EagerNet(kind, sd, [256, 128], dev, lr, 1e-5)
        for _ in range(epochs):
            tb = [torch.as_tensor(b) for b in trl[f]]
            steps += len(tb)
            M.run_pass(args, net, train, tb, True, lr, 1e-5)
            M.run_pass(args, net, train, [torch.as_tensor(b) for b in evl[f]])
            for j, ts in enumerate(tests):
                M.run_pass(args, net, ts, [torch.as_tensor(b) for b in tel[j]])
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return dict(arm=arm, model_type=kind, setting=setting, lr=lr, test_sets=list(test_sets), folds=folds,
                epochs=epochs, train_steps=steps, wall_s=round(wall, 3), ms_per_epoch=round(1e3 * wall / (folds * epochs), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", default="ours,eager")
    ap.add_argument("--models", default="mlp,attention")
    ap.add_argument("--settings", default="default,run_release")
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--eager_folds", type=int, default=None, help="shorter runs for the eager arm")
    ap.add_argument("--eager_epochs", type=int, default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mer2023_train needs a GPU"
    dev = torch.device("cuda", 0)
    name, power = card()
    rows = []
    for arm in a.arms.split(","):
        folds = a.eager_folds if (arm == "eager" and a.eager_folds) else a.folds
        epochs = a.eager_epochs if (arm == "eager" and a.eager_epochs) else a.epochs
        for kind in a.models.split(","):
            for setting in a.settings.split(","):
                r = run(arm, kind, setting, folds, epochs, dev)
                r.update(gpu=name, power_limit=power)
                print(json.dumps(r), flush=True)
                rows.append(r)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
