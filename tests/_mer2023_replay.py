"""Replays of tests/golden/mer2023_baseline_golden.npz (tests/golden/make_golden_mer2023_baseline.py) through
mertools_b200.main_release_mer2023.main: the recorded initial-weight generator states, sampler orders and dropout
keep-masks are fed back, and what the trainer computes is compared with what the unmodified reference computed."""
import os
import random
import re
import types

import numpy as np
import torch

from mertools_b200 import main_release_mer2023 as M
from mertools_b200 import synthetic as S
from mertools_b200.fusion_mlp import param_shapes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mer2023_baseline_golden.npz")
N_PASSES = 5   # train, eval, test1, test2, test3 per epoch


def golden():
    return np.load(GOLDEN, allow_pickle=False)


class Replay:
    def __init__(self, g, tag, mask_device, mask_dtype):
        self.g, self.tag, self.ptr = g, tag, 0
        self.dev, self.dtype = mask_device, mask_dtype
        self.epochs = int(g["epochs"])
        self.n_per_batch = None
        self.losses, self.best, self.nets = [], [], []

    def init_rng(self, fold):
        return torch.from_numpy(self.g[f"{self.tag}_rng"][fold].copy())

    def order(self, fold, epoch, which):
        return self.g[f"{self.tag}_order{(fold * self.epochs + epoch) * 2 + (which == 'eval')}"]

    def masks(self, fold, epoch, batch):
        out = []
        for _ in range(self.n_per_batch):
            shape = tuple(int(s) for s in self.g[f"{self.tag}_mask{self.ptr}_shape"])
            bits = np.unpackbits(self.g[f"{self.tag}_mask{self.ptr}"])[:int(np.prod(shape))].reshape(shape)
            out.append(torch.from_numpy(bits.astype(np.float32)).to(self.dev, self.dtype))
            self.ptr += 1
        return out

    def on_fold(self, fold, test_save, best_index, net):
        self.best.append(best_index)


class LossTap:
    """Wraps a net: records every training step's loss."""

    def __init__(self, net, sink):
        self.net, self.sink = net, sink

    def train_step(self, *a, **k):
        out = self.net.train_step(*a, **k)
        self.sink.append(float(out[0][2]))
        return out

    def __call__(self, *a):
        return self.net(*a)


def run(tag, work, make_net=None, device=None, mask_device="cpu", mask_dtype=torch.bool):
    """Writes the golden's corpus and label files under ``work``, replays configuration ``tag`` ('mlp' | 'att') and
    returns (replay, written paths, folder_save, name_time, args)."""
    g = golden()
    label_path, feats = S.write_mer2023_corpus(work, n_train=int(g["n_train"]), n_test=int(g["n_test"]),
                                               seed=int(g["seed"]), dims=tuple(int(d) for d in g["dims"]),
                                               numeric_val=True)
    os.makedirs(os.path.join(work, "dataset-release"), exist_ok=True)
    for ts in ("test1", "test3"):
        with open(os.path.join(work, "dataset-release", f"{ts}-label.csv"), "w") as fh:
            fh.write("\n".join(str(l) for l in g[f"label_{ts}"]) + "\n")
    argv = [str(a) for a in g[f"{tag}_argv"]]
    argv = [a if not a.startswith("--save_root=") else f"--save_root={work}/saved_{tag}" for a in argv]
    args = M.build_parser().parse_args(argv)
    rp = Replay(g, tag, mask_device, mask_dtype)
    n_layers = len(args.layers.split(","))
    rp.n_per_batch = n_layers * (1 if args.model_type == "mlp" else 4)
    cfg = types.SimpleNamespace(PATH_TO_LABEL={"MER2023": label_path}, PATH_TO_FEATURES={"MER2023": feats})
    if make_net is not None:
        inner = make_net
        make_net = lambda kind, dims, sd: LossTap(inner(kind, dims, sd), rp.losses)  # noqa: E731
    random.seed(int(g["seed"]))
    cwd = os.getcwd()
    os.chdir(work)
    try:
        written, folder_save, name_time = M.main(args, config=cfg, replay=rp, make_net=make_net, device=device)
    finally:
        os.chdir(cwd)
    return rp, written, folder_save, name_time, args


_NUM = re.compile(r"-?\d+\.\d+")


def same_name(got, ref, tol):
    """Result-file names: equal text, numbers within tol."""
    a, b = _NUM.split(got), _NUM.split(ref)
    assert a == b, (got, ref)
    for x, y in zip(_NUM.findall(got), _NUM.findall(ref)):
        assert abs(float(x) - float(y)) <= tol, (got, ref)


def check_replay(tag, rp, written, folder_save, name_time, args, work, tol):
    """Everything the golden recorded, with tolerance ``tol`` on computed values (absolute and relative)."""
    g = golden()
    ep = int(g["epochs"])
    close = lambda x, y, what: np.testing.assert_allclose(np.asarray(x, np.float64), np.asarray(y, np.float64),  # noqa: E731
                                                          rtol=tol, atol=tol, err_msg=f"{tag} {what}")
    # fold membership: the eval indices of each fold
    folds = _folds(g)
    for f in range(5):
        assert sorted(g[f"{tag}_order{f * ep * 2 + 1}"].tolist()) == folds[f], (tag, f)
    # every training step's loss, every pass's F1 / MSE
    close(rp.losses, g[f"{tag}_losses"], "train losses")
    n = 5 * ep * N_PASSES
    f1 = g[f"{tag}_f1"][:n].reshape(5, ep, N_PASSES)
    mse = g[f"{tag}_mse"][:n].reshape(5, ep, N_PASSES)
    best = [int(np.argmax(f1[f, :, 1] - 0.25 * mse[f, :, 1])) for f in range(5)]
    assert rp.best == best, (tag, rp.best, best)
    for f in range(5):
        fs = folder_save[f]
        for k in ("eval_names", "test1_names", "test2_names", "test3_names"):
            assert list(fs[k]) == list(g[f"{tag}_fold{f}_{k}"]), (tag, f, k)
        for k in ("eval_emoprobs", "eval_valpreds", "test1_emoprobs", "test1_valpreds", "test2_emoprobs",
                  "test2_valpreds", "test3_emoprobs", "test3_valpreds"):
            close(fs[k], g[f"{tag}_fold{f}_{k}"], f"fold {f} {k}")
        close([fs["eval_fscore"], fs["eval_valmse"]], [f1[f, best[f], 1], mse[f, best[f], 1]], f"fold {f} eval metrics")
    # state_dict names and shapes
    shapes = param_shapes(args.model_type, *[int(d) for d in g["dims"]], args.layers)
    assert list(shapes) == list(g[f"{tag}_sd_names"])
    assert [str(tuple(s)) for s in shapes.values()] == list(g[f"{tag}_sd_shapes"])
    # output files and the submission CSVs
    root = f"{work}/saved_{tag}-trimodal"
    got = sorted(os.path.relpath(p, root).replace(str(name_time), "TIME") for p in written)
    for a, b in zip(got, sorted(str(s) for s in g[f"{tag}_saved"])):
        same_name(a, b, 2e-4 if tol > 1e-6 else 0.0)
    assert len(got) == len(g[f"{tag}_saved"])
    for ts in ("test1", "test2", "test3"):
        ref = [l.split(",") for l in g[f"{tag}_csv_{ts}"]]
        mine = [l.split(",") for l in open(f"{root}/prediction/{ts}-pred-{name_time}.csv").read().splitlines()]
        assert ref[0] == mine[0] == ["name", "discrete", "valence"]
        assert [r[:2] for r in mine[1:]] == [r[:2] for r in ref[1:]], (tag, ts)
        close([float(r[2]) for r in mine[1:]], [float(r[2]) for r in ref[1:]], f"{ts} csv valence")


def _folds(g):
    random.seed(int(g["seed"]))
    return [sorted(int(i) for i in ev) for _, ev in M.random_split_indexes(int(g["n_train"]), 5)]
