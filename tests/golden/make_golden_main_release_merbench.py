"""Golden of the UNMODIFIED MERBench trainer on the corpora beyond MER2023: ``runpy`` of
/root/reference/MERBench/main-release.py on synthetic corpora of synthetic.write_merbench_corpus (label files in the
formats of toolkit/preprocess/{cmumosi,sims,iemocap,meld}.py) for 3 epochs with dropout 0 (the only RNG-free setting:
the reference draws its dropout masks from torch's generator), batch 32, hidden 64, in six configurations:
    cmumosi_utt        --dataset CMUMOSI (regression-only head, train / val / test, sequential train loader);
    sims_frm_align     --dataset SIMS --feat_type frm_align (the LSTM net on frame-level features);
    iemocapfour_utt    --dataset IEMOCAPFour (leave-one-session-out folds, no test set);
    meld_utt           --dataset MELD (7 classes, train / val / test);
    crossdim_sims_cmumosi      --train_dataset SIMS --test_dataset CMUMOSI (SIMS valences x 3);
    crossdis_iemocapfour_meld  --train_dataset IEMOCAPFour --test_dataset MELD (the four shared emotions).

Run once in the build container (needs /root/reference; NOT on the GPU box):
    python tests/golden/make_golden_main_release_merbench.py
Writes tests/golden/main_release_merbench_golden.npz, keys prefixed by the configuration name: fold membership (train
and eval names of epoch 0 per fold, in the order the reference's loaders visited them), train / eval / test loss of every
epoch of every fold, the best epoch of each fold with its eval scores, and the result-file names without their
wall-clock suffix.

Harness only -- no reference source is copied or edited.  The stubs and observers are those of
make_golden_main_release.py (via make_golden_main_release_mer2026._stubs); config.PATH_TO_LABEL / PATH_TO_FEATURES of
every corpus are patched to the synthetic corpora.
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
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, OUT)
REF = "/root/reference/MERBench"
SEED = 0
EPOCHS = 3
HYPER = "attention:\n  hidden_dim: 64\n  dropout: 0.0\n  grad_clip: -1.0\n  lr: 0.001\n"
UTT = ["--feat_type=utt", "--audio_feature=synA-UTT", "--text_feature=synT-UTT", "--video_feature=synV-UTT"]
FRA = ["--feat_type=frm_align", "--audio_feature=synA-FRA", "--text_feature=synT-FRA", "--video_feature=synV-FRA"]
CONFIGS = {
    "cmumosi_utt": ["--dataset=CMUMOSI", *UTT],
    "sims_frm_align": ["--dataset=SIMS", *FRA],
    "iemocapfour_utt": ["--dataset=IEMOCAPFour", *UTT],
    "meld_utt": ["--dataset=MELD", *UTT],
    "crossdim_sims_cmumosi": ["--train_dataset=SIMS", "--test_dataset=CMUMOSI", *UTT],
    "crossdis_iemocapfour_meld": ["--train_dataset=IEMOCAPFour", "--test_dataset=MELD", *UTT],
}
# corpus -> clips per split (IEMOCAP: whole_corpus) and its seed
CORPORA = {"CMUMOSI": ((40, 12, 12), 1), "SIMS": ((40, 12, 12), 2), "IEMOCAPFour": ((50,), 3), "MELD": ((40, 12, 12), 4)}

from mertools_b200 import synthetic as S  # noqa: E402


def write_corpora(work):
    """Every corpus of CORPORA under work/<name>/ -> {name: (label_path, feature_root)}."""
    return {ds: S.write_merbench_corpus(os.path.join(work, ds), ds, n=n, seed=seed, frame_level=ds == "SIMS")
            for ds, (n, seed) in CORPORA.items()}


def run(name, argv, work, corpora, hyper):
    import config as ref_config  # the reference's own config module (paths patched below)
    for ds, (lp, fr) in corpora.items():
        ref_config.PATH_TO_LABEL[ds] = lp
        ref_config.PATH_TO_FEATURES[ds] = fr
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
    sys.argv = ["main-release.py", "--model=attention", *argv, f"--hyper_path={hyper}", f"--epochs={EPOCHS}",
                "--batch_size=32", f"--save_root={work}/saved_{name}", "--gpu=0"]
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
    folds = len(g["folder_save"])
    n_tests = len(g["test_loaders"])
    assert len(saved) == 1 + n_tests, saved
    out = {
        "folds": folds,
        "train_loss": np.array(seen["train_loss"], np.float64).reshape(folds, EPOCHS),
        "eval_loss": np.array(seen["eval_loss"], np.float64).reshape(folds, EPOCHS),
        # the reference stores test losses fold by fold, epoch by epoch, test set by test set
        "test_loss": np.array(seen["test_loss"], np.float64).reshape(folds, EPOCHS, n_tests).transpose(2, 0, 1),
        "saved": np.array(saved),
        "best_index": np.array([int(l.split("best_index: ")[1].split(",")[0]) for l in lines if "best_index:" in l]),
        "feat_dims": np.array([g["args"].audio_dim, g["args"].text_dim, g["args"].video_dim]),
        "output_dims": np.array([g["args"].output_dim1, g["args"].output_dim2]),
    }
    for f in range(folds):
        out[f"fold{f}_train_names_epoch0"] = np.array(seen["train_names"][f * EPOCHS])
        out[f"fold{f}_eval_names_epoch0"] = np.array(seen["eval_names"][f * EPOCHS])
        best = g["folder_save"][f]
        for k in ("eval_emofscore", "eval_emoacc", "eval_loss"):
            out[f"fold{f}_{k}"] = float(best[k])
    print(name, "\n  ".join([""] + saved), "\n  train_loss", out["train_loss"][0])
    return {f"{name}_{k}": v for k, v in out.items()}


def main():
    from make_golden_main_release_mer2026 import _stubs
    work = tempfile.mkdtemp(prefix="mer_golden_mrb_")
    corpora = write_corpora(work)
    hyper = os.path.join(work, "hyper.yaml")
    open(hyper, "w").write(HYPER)
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    _stubs()
    out = dict(seed=SEED, epochs=EPOCHS, hyper=HYPER, configs=np.array(list(CONFIGS)))
    try:
        for name, argv in CONFIGS.items():
            out.update(run(name, argv, work, corpora, hyper))
    finally:
        os.chdir(cwd)
    np.savez_compressed(os.path.join(OUT, "main_release_merbench_golden.npz"), **out)


if __name__ == "__main__":
    main()
