"""Golden of the UNMODIFIED MER2023 baseline trainer: ``runpy`` of MER2023/main-release.py on a synthetic MER2023-format
corpus (45 train clips, 3 x 10 test clips, every valence numeric, A / T / V widths 10 / 12 / 7 -- two of them not a
multiple of 4) for 3 epochs over the 5 folds with ``--test_sets test1,test2,test3``, in two configurations:
``--model_type mlp`` with the default ``--layers 256,128`` and ``--model_type attention --layers 24,16,8``.  The
working directory holds ``dataset-release/test1-label.csv`` and ``test3-label.csv`` (a subset), so both report
functions run; test2 has no label file ('nores').

Run once where the reference tree is available (CPU only; not on the GPU machine):
    python tests/golden/make_golden_mer2023_baseline.py /path/to/MER2023
Writes tests/golden/mer2023_baseline_golden.npz.

Harness only -- no reference source is copied or edited.  The script seeds nothing, so ``random``, ``numpy`` and
``torch`` are seeded first.  Stubs as in make_golden_main_release.py: ``torch.cuda.set_device``, ``Tensor.cuda`` and
``Module.cuda`` are no-ops, ``multiprocessing.Pool`` is a thread pool.  Pass-through observers record what the script
computes:
  * ``nn.Dropout.forward``: the keep-mask of every call (torch's CPU dropout is ``x * bernoulli(1 - p) / (1 - p)``;
    the observer re-draws the same Bernoulli tensor from the generator state the call started from, checks the
    output against it and leaves the generator where the call left it);
  * ``SubsetRandomSampler.__iter__``: every sample order the train and eval loaders visit;
  * ``nn.Linear.__init__``: torch's generator state before the first Linear of each fold's model;
  * ``Tensor.backward``: every training batch's loss;
  * ``sklearn.metrics.f1_score`` / ``mean_squared_error``: every pass's F1 and MSE.
"""
import contextlib
import io
import os
import random
import runpy
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.dirname(os.path.abspath(__file__))
SEED, EPOCHS = 0, 3
DIMS = (10, 12, 7)
N_TRAIN, N_TEST = 45, 10
CONFIGS = {"mlp": ["--model_type=mlp"], "att": ["--model_type=attention", "--layers=24,16,8"]}

from mertools_b200 import synthetic as S  # noqa: E402


def run(ref, tag, extra, work, label_path, feats):
    import multiprocessing
    import multiprocessing.pool

    import sklearn.metrics as skm
    from torch.utils.data.sampler import SubsetRandomSampler
    torch.cuda.set_device = lambda *a, **k: None
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    multiprocessing.Pool = lambda processes=None: multiprocessing.pool.ThreadPool(processes)
    sys.path.insert(0, ref)
    import config as ref_config
    ref_config.PATH_TO_LABEL["MER2023"] = label_path
    ref_config.PATH_TO_FEATURES["MER2023"] = feats

    seen = dict(masks=[], orders=[], rng=[], losses=[], f1=[], mse=[])
    state = dict(new_model=True)
    drop_fwd, lin_init, sampler_iter = torch.nn.Dropout.forward, torch.nn.Linear.__init__, SubsetRandomSampler.__iter__
    backward, f1_score, mse = torch.Tensor.backward, skm.f1_score, skm.mean_squared_error

    def drop_obs(self, x):
        if not self.training or self.p == 0:
            return drop_fwd(self, x)
        before = torch.get_rng_state()
        y = drop_fwd(self, x)
        after = torch.get_rng_state()
        torch.set_rng_state(before)
        keep = torch.empty_like(x).bernoulli_(1 - self.p)
        torch.set_rng_state(after)
        assert torch.equal(y, x * keep.div(1 - self.p)), "dropout is not x * bernoulli(1 - p) / (1 - p)"
        seen["masks"].append(keep.bool().numpy())
        return y

    def lin_obs(self, *a, **k):
        if state["new_model"]:
            seen["rng"].append(torch.get_rng_state().numpy().copy())
            state["new_model"] = False
        return lin_init(self, *a, **k)

    def sampler_obs(self):
        order = list(sampler_iter(self))
        seen["orders"].append(np.array(order, np.int64))
        state["new_model"] = True      # the next Linear built belongs to the next fold's model
        return iter(order)

    def backward_obs(self, *a, **k):
        seen["losses"].append(float(self.detach()))
        return backward(self, *a, **k)

    def f1_obs(*a, **k):
        r = f1_score(*a, **k)
        seen["f1"].append(float(r))
        return r

    def mse_obs(*a, **k):
        r = mse(*a, **k)
        seen["mse"].append(float(r))
        return r

    torch.nn.Dropout.forward, torch.nn.Linear.__init__, SubsetRandomSampler.__iter__ = drop_obs, lin_obs, sampler_obs
    torch.Tensor.backward, skm.f1_score, skm.mean_squared_error = backward_obs, f1_obs, mse_obs
    argv = ["--dataset=MER2023", "--audio_feature=synA-UTT", "--text_feature=synT-UTT", "--video_feature=synV-UTT",
            "--test_sets=test1,test2,test3", f"--epochs={EPOCHS}", f"--save_root={work}/saved_{tag}"] + extra
    sys.argv = ["main-release.py"] + argv
    random.seed(SEED)
    np.random.seed(SEED)
    torch.manual_seed(SEED)
    buf = io.StringIO()
    cwd = os.getcwd()
    os.chdir(work)
    try:
        with contextlib.redirect_stdout(buf):
            g = runpy.run_path(os.path.join(ref, "main-release.py"), run_name="__main__")
    finally:
        os.chdir(cwd)
        torch.nn.Dropout.forward, torch.nn.Linear.__init__, SubsetRandomSampler.__iter__ = drop_fwd, lin_init, \
            sampler_iter
        torch.Tensor.backward, skm.f1_score, skm.mean_squared_error = backward, f1_score, mse
    lines = buf.getvalue().splitlines()
    name_time = str(g["name_time"])
    saved = sorted(os.path.relpath(os.path.join(d, f), f"{work}/saved_{tag}-trimodal").replace(name_time, "TIME")
                   for d, _, fs in os.walk(f"{work}/saved_{tag}-trimodal") for f in fs)
    out = {f"{tag}_argv": np.array(argv), f"{tag}_saved": np.array(saved),
           f"{tag}_rng": np.stack(seen["rng"]), f"{tag}_losses": np.array(seen["losses"]),
           f"{tag}_f1": np.array(seen["f1"]), f"{tag}_mse": np.array(seen["mse"]),
           f"{tag}_epoch_lines": np.array([l for l in lines if l.startswith("epoch:")])}
    assert len(seen["rng"]) == 5 and len(seen["orders"]) == 5 * EPOCHS * 2, (len(seen["rng"]), len(seen["orders"]))
    for i, o in enumerate(seen["orders"]):
        out[f"{tag}_order{i}"] = o
    out[f"{tag}_n_masks"] = np.array(len(seen["masks"]))
    for i, m in enumerate(seen["masks"]):
        out[f"{tag}_mask{i}_shape"] = np.array(m.shape)
        out[f"{tag}_mask{i}"] = np.packbits(m.reshape(-1))
    for f, best in enumerate(g["folder_save"]):
        for k, v in best.items():
            out[f"{tag}_fold{f}_{k}"] = np.asarray(v) if k.endswith("names") else np.asarray(v, np.float32)
    sd = g["model"].state_dict()
    out[f"{tag}_sd_names"] = np.array(list(sd))
    out[f"{tag}_sd_shapes"] = np.array([str(tuple(v.shape)) for v in sd.values()])
    pred = os.path.join(f"{work}/saved_{tag}-trimodal", "prediction")
    for f in sorted(os.listdir(pred)):
        out[f"{tag}_csv_{f.split('-pred-')[0]}"] = np.array(open(os.path.join(pred, f)).read().splitlines())
    sys.path.remove(ref)
    sys.modules.pop("config", None)
    return out


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/MER2023"
    work = tempfile.mkdtemp(prefix="mer_golden_mer2023_")
    label_path, feats = S.write_mer2023_corpus(work, n_train=N_TRAIN, n_test=N_TEST, seed=SEED, dims=DIMS,
                                               numeric_val=True)
    # the challenge's label files for the report functions: all of test1, half of test3
    rng = np.random.default_rng(SEED + 1)
    os.makedirs(os.path.join(work, "dataset-release"))
    for ts, n in (("test1", N_TEST), ("test3", N_TEST // 2)):
        with open(os.path.join(work, "dataset-release", f"{ts}-label.csv"), "w") as fh:
            fh.write("name,discrete,valence\n")
            for i in range(n):
                fh.write(f"{ts}_{i:04d},{S.EMOS_MER[int(rng.integers(0, 6))]},{float(rng.uniform(-3, 3))!r}\n")
    out = dict(seed=SEED, epochs=EPOCHS, dims=np.array(DIMS), n_train=N_TRAIN, n_test=N_TEST)
    for ts in ("test1", "test3"):
        out[f"label_{ts}"] = np.array(open(os.path.join(work, "dataset-release", f"{ts}-label.csv")).read()
                                      .splitlines())
    for tag, extra in CONFIGS.items():
        out.update(run(ref, tag, extra, work, label_path, feats))
    np.savez_compressed(os.path.join(OUT, "mer2023_baseline_golden.npz"), **out)
    for tag in CONFIGS:
        print(tag, "losses", len(out[f"{tag}_losses"]), "masks", int(out[f"{tag}_n_masks"]), out[f"{tag}_saved"])


if __name__ == "__main__":
    main()
