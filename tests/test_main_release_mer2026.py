"""main_release for MER2024 / MER2025 / MER2026 (CPU): the corpus' label reader, top-N feature selection, result-file
names and cv strings, and a CPU replay through oracle/fusion.py of the golden runs of the unmodified MER2026 trainer
(tests/golden/make_golden_main_release_mer2026.py)."""
import os
import random
import types

import numpy as np
import pytest
import torch

from mertools_b200 import fusion as FU
from mertools_b200 import main_release as MR
from mertools_b200 import synthetic as S
from oracle import fusion as OF

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "main_release_mer2026_golden.npz")


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("mer2026"))
    label_path, feats = S.write_mer2026_corpus(root, seed=0)
    return types.SimpleNamespace(PATH_TO_LABEL={"MER2026": label_path}, PATH_TO_FEATURES={"MER2026": feats})


@pytest.mark.parametrize("dataset", MR.EMO_CORPORA)
def test_label_reader_emotion_only_corpora(corpus, dataset):
    path = corpus.PATH_TO_LABEL["MER2026"]
    names, labels = MR.read_names_labels(path, "train", dataset=dataset)
    raw = np.load(path, allow_pickle=True)["train_corpus"].tolist()
    assert names == list(raw) and len(names) == 80
    assert labels == [{"emo": MR.EMO2IDX[raw[n]["emo"]], "val": -10} for n in names]   # mer2026.py:92-94
    n1, _ = MR.read_names_labels(path, "test1", dataset=dataset)
    assert len(n1) == 20
    assert len(MR.read_names_labels(path, "train", debug=True, dataset=dataset)[0]) == 80
    for dt in ("test2", "test3"):      # one test set only (mer2026.py:85)
        with pytest.raises(AssertionError):
            MR.read_names_labels(path, dt, dataset=dataset)


def test_label_reader_mer2023_unchanged(tmp_path):
    label_path, _ = S.write_mer2023_corpus(str(tmp_path))
    names, labels = MR.read_names_labels(label_path, "train")
    assert labels[0]["val"] == -10 and labels[1]["val"] != -10 and len(MR.read_names_labels(label_path, "test3")[0]) == 8


@pytest.mark.parametrize("dataset", MR.EMO_CORPORA)
@pytest.mark.parametrize("modality", ["AVT", "AV", "AT", "VT"])
@pytest.mark.parametrize("topn", [1, 2, 3, 4, 5, 6])
def test_topn_selection(tmp_path, dataset, modality, topn):
    """feat_data_topn.py:16-31: the last n of each of the three lists, `<dir>_UTT` when that directory exists."""
    ranks = MR.RANK_LISTS[dataset]
    lists = [ranks[w] for w in MR.FUSION_MODALITIES[modality]]
    if any(len(l) < topn for l in lists):      # MER2026's text list has 4 entries, MER2025's 5
        with pytest.raises(AssertionError):
            MR.topn_feature_names(dataset, topn, modality, str(tmp_path))
        return
    expect = [n for l in lists for n in l[-topn:]]
    underscore = set(expect[::2])              # half of them exist as <dir>_UTT
    for n in underscore:
        os.makedirs(tmp_path / f"{MR.FEATNAME_DIRS[n]}_UTT", exist_ok=True)
    got = MR.topn_feature_names(dataset, topn, modality, str(tmp_path))
    assert len(got) == 3 * topn
    assert got == [MR.FEATNAME_DIRS[n] + ("_UTT" if n in underscore else "-UTT") for n in expect]


def test_topn_lists_pinned():
    """The modality strings take three lists, not one per modality (feat_data_topn.py:17-24), and every ranked name
    has a feature directory."""
    assert MR.FUSION_MODALITIES == {"AVT": ("audio", "text", "image"), "AT": ("audio", "text", "text"),
                                    "AV": ("audio", "image", "image"), "VT": ("text", "text", "image")}
    assert MR.RANK_LISTS["MER2026"]["audio"][-2:] == ["HUBERT-large", "HUBERT-base"]
    assert MR.RANK_LISTS["MER2024"]["image"][-1] == "CLIP-large" and len(MR.RANK_LISTS["MER2024"]["text"]) == 15
    used = {n for r in MR.RANK_LISTS.values() for l in r.values() for n in l}
    assert used == set(MR.FEATNAME_DIRS)
    assert MR.func_name_conversion("VideoMAE-base (MER2023)", "/nonexistent") == "videomae-base-K400-mer2023-299-UTT"


def test_cv_strings_and_results():
    """metric.py:35-54 prints the present keys only; mer2026.py:132-145 reports f1 and acc."""
    fs = [dict(eval_emofscore=0.5, eval_emoacc=0.25), dict(eval_emofscore=0.25, eval_emoacc=0.5)]
    assert MR.gain_cv_results(fs) == "f1:0.3750_acc:0.3750"
    fs = [dict(eval_emofscore=0.5, eval_emoacc=0.25, eval_valmse=2.0)]
    assert MR.gain_cv_results(fs) == "f1:0.5000_acc:0.2500_val:2.0000"
    probs = np.eye(6, dtype=np.float32)[[0, 1, 2, 2]]
    res, s = FU.mer2026_calculate_results(probs, np.array([0, 1, 2, 3]), [], [])
    assert s == "f1:0.6667_acc:0.7500" and set(res) == {"emoprobs", "emolabels", "emoacc", "emofscore"}
    assert MR.corpus_calculate_results("MER2026") is FU.mer2026_calculate_results
    assert MR.corpus_calculate_results("MER2023") is FU.mer2023_calculate_results


def test_reference_init_topn_draws_like_the_reference():
    """torch's own constructors in Attention_TOPN.__init__ order: the same values and the same generator state as
    building the nn.Linear modules by hand in that order; fc_out_2 is [0, H] / [0] at output_dim2 = 0."""
    dims, H = [5, 7, 3], 4
    torch.manual_seed(1)
    sd = FU.reference_init_topn(dims, H, 6, 0)
    after = torch.rand(1)
    torch.manual_seed(1)
    ref = {}
    for e, d in [(f"encoder{i}", d) for i, d in enumerate(dims)] + [("attention_mlp", H * len(dims))]:
        for l, k in (("linear_1", d), ("linear_2", H), ("linear_3", H)):
            ref.update({f"{e}.{l}.{n}": v for n, v in torch.nn.Linear(k, H).state_dict().items()})
    for l, o in (("fc_att", len(dims)), ("fc_out_1", 6), ("fc_out_2", 0)):
        ref.update({f"{l}.{n}": v for n, v in torch.nn.Linear(H, o).state_dict().items()})
    assert list(sd) == list(ref) and all(torch.equal(sd[k], ref[k]) for k in sd)
    assert torch.equal(after, torch.rand(1))
    assert sd["fc_out_2.weight"].shape == (0, H) and sd["fc_out_2.bias"].shape == (0,)


# ---- CPU replay of the golden runs ------------------------------------------------------------------------------------
def _replay(g, cfg_name, corpus):
    """The mirror's host logic (label reader, top-N selection, fold split, loaders, initial weights) driving the
    oracle's fp32 CPU trainer, as the unmodified script ran (dropout 0, emotion-only head, CE loss)."""
    pre = f"{cfg_name}_"
    argv = {"attention": dict(model="attention"), "topn2_avt": dict(model="attention_topn", modality="AVT"),
            "topn2_at": dict(model="attention_topn", modality="AT")}[cfg_name]
    torch.manual_seed(int(g["seed"]))
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    root = corpus.PATH_TO_FEATURES["MER2026"]
    if argv["model"] == "attention":
        fnames = ["chinese-hubert-base-UTT"] * 3
    else:
        fnames = MR.topn_feature_names("MER2026", 2, argv["modality"], root)
    lp = corpus.PATH_TO_LABEL["MER2026"]
    names, labels = MR.read_names_labels(lp, "train", dataset="MER2026")
    tnames, tlabels = MR.read_names_labels(lp, "test1", dataset="MER2026")
    X = [torch.from_numpy(np.stack([MR.read_utt_feature(os.path.join(root, f), n) for n in names]).astype(np.float32))
         for f in fnames]
    XT = [torch.from_numpy(np.stack([MR.read_utt_feature(os.path.join(root, f), n) for n in tnames]).astype(np.float32))
          for f in fnames]
    emo = torch.tensor([l["emo"] for l in labels])
    temo = torch.tensor([l["emo"] for l in tlabels])
    folds = MR.random_split_indexes(len(names), 5)
    trl, evl, tel = MR.get_loaders(len(names), folds, [len(tnames)], 32)
    dims = [int(x.shape[1]) for x in X]
    assert dims == list(g[pre + "feat_dims"])
    E = int(g["epochs"])
    out = dict(train=np.zeros((5, E)), eval=np.zeros((5, E)), test=np.zeros((5, E)), best=[], names=[], tnames=[])

    def fwd(sd, xs):
        if argv["model"] == "attention":
            return OF.attention_forward(sd, *xs)[1]
        return OF.attention_topn_forward(sd, xs)[1]

    def evaluate(sd, xs_all, y_all, loader):
        losses, probs, order = [], [], []
        with torch.no_grad():
            for b in loader:
                eo = fwd(sd, [x[b] for x in xs_all])
                losses.append(float(OF.losses(eo, torch.zeros(len(b), 0), y_all[b], torch.zeros(len(b), 0))[0]))
                probs.append(eo.numpy())
                order += b.tolist()
        probs = np.concatenate(probs)
        f1 = FU.mer2026_calculate_results(probs, y_all[order].numpy())[0]["emofscore"]
        return np.mean(losses), f1, order

    for f in range(5):
        if argv["model"] == "attention":
            sd = FU.reference_init("utt", *dims, 64, 6, 0)
        else:
            sd = FU.reference_init_topn(dims, 64, 6, 0)
        tr = OF.Trainer(sd, lr=1e-3, l2=1e-5)
        metrics = []
        for ep in range(E):
            losses, order = [], []
            for b in trl[f]:
                xs = [x[b] for x in X]
                args = (xs, None, None) if argv["model"] != "attention" else tuple(xs)
                ce, _, _, _, _, _ = tr.step(*args, emo[b], torch.zeros(len(b), 0))
                losses.append(ce)
                order += b.tolist()
            out["train"][f, ep] = np.mean(losses)
            out["eval"][f, ep], f1, eorder = evaluate(tr.sd, X, emo, evl[f])
            out["test"][f, ep], _, _ = evaluate(tr.sd, XT, temo, tel[0])
            metrics.append(f1)
            if ep == 0:
                out["names"].append([names[i] for i in eorder])
                out["tnames"].append([names[i] for i in order])
        out["best"].append(int(np.argmax(metrics)))
    return out


@pytest.mark.parametrize("cfg_name", ["attention", "topn2_avt", "topn2_at"])
def test_cpu_replay_of_the_golden(corpus, cfg_name):
    g = np.load(GOLDEN)
    pre = f"{cfg_name}_"
    r = _replay(g, cfg_name, corpus)
    for f in range(5):
        assert r["names"][f] == list(g[f"{pre}fold{f}_eval_names_epoch0"]), f"fold {f}: eval split / order"
        assert r["tnames"][f] == list(g[f"{pre}fold{f}_train_names_epoch0"]), f"fold {f}: train order"
    assert r["best"] == list(g[pre + "best_index"])
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()  # noqa: E731
    assert rel(r["train"], g[pre + "train_loss"]) < 1e-5
    assert rel(r["eval"], g[pre + "eval_loss"]) < 1e-5
    assert rel(r["test"], g[pre + "test_loss"][0]) < 1e-5
