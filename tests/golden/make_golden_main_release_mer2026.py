"""Golden of the UNMODIFIED MER2026 Track 1 trainer: ``runpy`` of /root/reference/MER2026/MER2026_Track1/main-release.py
on the synthetic corpus of synthetic.write_mer2026_corpus (80 train clips, 20 test1 clips, 5 folds, batch 32) for 3
epochs with dropout 0 (the only RNG-free setting: the reference draws its dropout masks from torch's generator), in
three configurations:
    attention   --model attention, one feature for A / T / V (as run-unimodal.sh runs it);
    topn2_avt   --model attention_topn --fusion_topn 2 --fusion_modality AVT (N = 6);
    topn2_at    --model attention_topn --fusion_topn 2 --fusion_modality AT (text features twice).

Run once in the build container (needs /root/reference; NOT on the GPU box):
    python tests/golden/make_golden_main_release_mer2026.py
Writes tests/golden/main_release_mer2026_golden.npz, keys prefixed by the configuration name: fold membership (train and
eval names of epoch 0 per fold, in the order the reference's SubsetRandomSampler visited them), train / eval / test1
loss of every epoch of every fold, the best epoch of each fold with its eval / test1 emotion scores, and the
result-file names without their wall-clock suffix.

Harness only -- no reference source is copied or edited.  The stubs and observers are those of
make_golden_main_release.py; in addition config.PATH_TO_FEATURES['MER2026'] / PATH_TO_LABEL['MER2026'] are patched
to the synthetic corpus.  The MER2026 toolkit imports, at module level, libraries that only its preprocessing and
end-to-end paths call (OpenCV, torchaudio, matplotlib, the OpenAI client, the AffectGPT / ImageBind audio loader of
read_data.py); each of those that does not import here is served by an inert stand-in module (every attribute and
every call is another inert object; matplotlib.use('Agg') runs at import time).
"""
import contextlib
import importlib
import io
import os
import random
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference/MER2026/MER2026_Track1"
OUT = os.path.dirname(os.path.abspath(__file__))
SEED = 0
EPOCHS = 3
HYPER = ("attention:\n  hidden_dim: 64\n  dropout: 0.0\n  grad_clip: -1.0\n  lr: 0.001\n"
         "attention_topn:\n  hidden_dim: 64\n  dropout: 0.0\n  grad_clip: -1.0\n  lr: 0.001\n")
UNIMODAL = "chinese-hubert-base-UTT"
CONFIGS = {
    "attention": ["--model=attention", f"--audio_feature={UNIMODAL}", f"--text_feature={UNIMODAL}",
                  f"--video_feature={UNIMODAL}"],
    "topn2_avt": ["--model=attention_topn", "--fusion_topn=2", "--fusion_modality=AVT"],
    "topn2_at": ["--model=attention_topn", "--fusion_topn=2", "--fusion_modality=AT"],
}

from mertools_b200 import synthetic as S  # noqa: E402


def _stubs():
    import yaml
    oc = types.ModuleType("omegaconf")
    oc.OmegaConf = types.SimpleNamespace(load=lambda p: yaml.safe_load(open(p)))
    sys.modules["omegaconf"] = oc
    thop = types.ModuleType("thop")
    thop.profile = lambda *a, **k: (0, 0)
    sys.modules["thop"] = thop
    torch.cuda.set_device = lambda *a, **k: None
    torch.cuda.empty_cache = lambda: None
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    import multiprocessing
    import multiprocessing.pool
    multiprocessing.Pool = lambda processes=None: multiprocessing.pool.ThreadPool(processes)
    for name in STANDINS:
        try:
            importlib.import_module(name)
        except Exception:  # noqa: BLE001 -- a missing library, or a dependency of one
            sys.meta_path.insert(0, _StandInFinder(name))


STANDINS = ("cv2", "torchaudio", "matplotlib", "openai", "toolkit.models.modules.affectgpt.models.ImageBind.data")


class _Inert:
    def __init__(self, name):
        self._name = name

    def __call__(self, *a, **k):
        return _Inert(f"{self._name}()")

    def __getattr__(self, k):
        return _Inert(f"{self._name}.{k}")

    def __mro_entries__(self, bases):
        return (object,)


class _StandInModule(types.ModuleType):
    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return _Inert(f"{self.__name__}.{k}")


class _StandInFinder:
    """Serves `name` and its submodules as _StandInModule packages."""

    def __init__(self, name):
        self.name = name

    def find_spec(self, fullname, path=None, target=None):
        import importlib.machinery
        if fullname == self.name or fullname.startswith(self.name + "."):
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StandInModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def run(name, argv, work, label_path, feats, hyper):
    import config as ref_config  # the reference's own config module (paths patched below)
    ref_config.PATH_TO_LABEL["MER2026"] = label_path
    ref_config.PATH_TO_FEATURES["MER2026"] = feats
    import toolkit.utils.functions as F
    import toolkit.utils.metric as M
    seen = dict(train_loss=[], eval_loss=[], test_loss=[], eval_names=[], train_names=[])
    gain, update = M.gain_metric_from_results, F.func_update_storage
    calls = [0]

    def gain_observer(res, metric_name="emoval"):
        key = "train" if calls[0] % 2 == 0 else "eval"
        calls[0] += 1
        seen[f"{key}_loss"].append(float(res["loss"]))
        seen[f"{key}_names"].append(list(res["names"]))
        return gain(res, metric_name)

    def update_observer(inputs, prefix, outputs):
        if prefix.startswith("test"):
            seen["test_loss"].append(float(inputs["loss"]))
        return update(inputs, prefix, outputs)

    M.gain_metric_from_results = gain_observer
    F.func_update_storage = update_observer
    sys.argv = ["main-release.py", "--feat_type=utt", "--dataset=MER2026", *argv, f"--hyper_path={hyper}",
                f"--epochs={EPOCHS}", f"--save_root={work}/saved_{name}", "--gpu=0"]
    torch.manual_seed(SEED)
    random.seed(SEED)
    np.random.seed(SEED)
    buf = io.StringIO()
    try:
        with contextlib.redirect_stdout(buf):
            g = runpy.run_path("main-release.py", run_name="__main__")
    finally:
        M.gain_metric_from_results, F.func_update_storage = gain, update
    lines = buf.getvalue().splitlines()
    saved = [os.path.basename(l.split("save results in ")[1]) for l in lines if l.startswith("save results in ")]
    name_time = str(g["name_time"])
    saved = [s.replace("_" + name_time + ".npz", "") for s in saved]  # drop the wall-clock suffix
    assert len(saved) == 2, saved
    out = {
        "train_loss": np.array(seen["train_loss"], np.float64).reshape(5, EPOCHS),
        "eval_loss": np.array(seen["eval_loss"], np.float64).reshape(5, EPOCHS),
        "test_loss": np.array(seen["test_loss"], np.float64).reshape(1, 5, EPOCHS),
        "saved": np.array(saved),
        "best_index": np.array([int(l.split("best_index: ")[1].split(",")[0]) for l in lines if "best_index:" in l]),
        "feat_dims": np.array(g["args"].audio_dim if isinstance(g["args"].audio_dim, list) else
                              [g["args"].audio_dim, g["args"].text_dim, g["args"].video_dim]),
    }
    for f in range(5):
        out[f"fold{f}_train_names_epoch0"] = np.array(seen["train_names"][f * EPOCHS])
        out[f"fold{f}_eval_names_epoch0"] = np.array(seen["eval_names"][f * EPOCHS])
        best = g["folder_save"][f]
        out[f"fold{f}_eval_names"] = np.array(best["eval_names"])
        for k in ("eval_emoprobs", "test1_emoprobs"):
            out[f"fold{f}_{k}"] = np.asarray(best[k], np.float32)
        for k in ("eval_emofscore", "eval_emoacc", "eval_loss"):
            out[f"fold{f}_{k}"] = float(best[k])
    print(name, "\n  ".join([""] + saved), "\n  train_loss", out["train_loss"][0])
    return {f"{name}_{k}": v for k, v in out.items()}


def main():
    work = tempfile.mkdtemp(prefix="mer_golden_mr26_")
    label_path, feats = S.write_mer2026_corpus(work, seed=SEED)
    hyper = os.path.join(work, "hyper.yaml")
    open(hyper, "w").write(HYPER)
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    _stubs()
    out = dict(seed=SEED, epochs=EPOCHS, hyper=HYPER, configs=np.array(list(CONFIGS)))
    try:
        for name, argv in CONFIGS.items():
            out.update(run(name, argv, work, label_path, feats, hyper))
    finally:
        os.chdir(cwd)
    np.savez_compressed(os.path.join(OUT, "main_release_mer2026_golden.npz"), **out)


if __name__ == "__main__":
    main()
