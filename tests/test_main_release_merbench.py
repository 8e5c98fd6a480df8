"""main_release for the MERBench corpora beyond MER2023 (CPU): label readers and the crossdis mapping, the SIMS x 3
scaling, the IEMOCAP session folds, loader order for every protocol, the acc-2 rule against sklearn, result names, and
a CPU replay through oracle/fusion.py of the golden runs of the unmodified MERBench trainer
(tests/golden/make_golden_main_release_merbench.py)."""
import argparse
import os
import random
import types

import numpy as np
import pytest
import torch
from sklearn.metrics import accuracy_score, f1_score

from mertools_b200 import fusion as FU
from mertools_b200 import main_release as MR
from mertools_b200 import synthetic as S
from oracle import fusion as OF

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "main_release_merbench_golden.npz")
# the corpora of make_golden_main_release_merbench.py: clips per split and seed
CORPORA = {"CMUMOSI": ((40, 12, 12), 1), "SIMS": ((40, 12, 12), 2), "IEMOCAPFour": ((50,), 3), "MELD": ((40, 12, 12), 4)}
ARGV = {
    "cmumosi_utt": dict(dataset="CMUMOSI", feat_type="utt"),
    "sims_frm_align": dict(dataset="SIMS", feat_type="frm_align"),
    "iemocapfour_utt": dict(dataset="IEMOCAPFour", feat_type="utt"),
    "meld_utt": dict(dataset="MELD", feat_type="utt"),
    "crossdim_sims_cmumosi": dict(train_dataset="SIMS", test_dataset="CMUMOSI", feat_type="utt"),
    "crossdis_iemocapfour_meld": dict(train_dataset="IEMOCAPFour", test_dataset="MELD", feat_type="utt"),
}


@pytest.fixture(scope="module")
def config(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("merbench"))
    paths = {ds: S.write_merbench_corpus(os.path.join(root, ds), ds, n=n, seed=seed, frame_level=ds == "SIMS")
             for ds, (n, seed) in CORPORA.items()}
    return types.SimpleNamespace(PATH_TO_LABEL={d: p[0] for d, p in paths.items()},
                                 PATH_TO_FEATURES={d: p[1] for d, p in paths.items()})


def _args(**kw):
    a = argparse.Namespace(dataset=None, train_dataset=None, test_dataset=None, model="attention", feat_type="utt",
                           feat_scale=1, debug=False, batch_size=32, num_workers=0, fusion_topn=None, e2e_name=None)
    a.__dict__.update(kw)
    if a.feat_type == "utt":
        a.audio_feature, a.text_feature, a.video_feature = "synA-UTT", "synT-UTT", "synV-UTT"
    else:
        a.audio_feature, a.text_feature, a.video_feature = "synA-FRA", "synT-FRA", "synV-FRA"
        a.feat_scale = 6 if a.feat_type == "frm_align" else 12
    return a


# ---- label readers ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dataset", ["CMUMOSI", "SIMS", "MELD"])
def test_label_reader_train_val_test(config, dataset):
    path = config.PATH_TO_LABEL[dataset]
    for dt, n in zip(("train", "val", "test"), CORPORA[dataset][0]):
        names, labels = MR.read_names_labels(path, dt, dataset=dataset)
        raw = np.load(path, allow_pickle=True)[f"{dt}_corpus"].tolist()
        assert names == list(raw) and len(names) == n
        assert labels == [{"emo": raw[k]["emo"], "val": raw[k]["val"]} for k in names]
        assert all(isinstance(l["emo"], int) for l in labels)
    with pytest.raises(AssertionError):
        MR.read_names_labels(path, "test1", dataset=dataset)


def test_label_reader_iemocap_whole(config):
    path = config.PATH_TO_LABEL["IEMOCAPFour"]
    assert os.path.basename(path) == "label_4way.npz"
    names, labels = MR.read_names_labels(path, "whole", dataset="IEMOCAPFour")
    raw = np.load(path, allow_pickle=True)["whole_corpus"].tolist()
    assert names == list(raw) and len(names) == 50 and {l["emo"] for l in labels} <= {0, 1, 2, 3}
    assert MR.read_names_labels(path, "whole", debug=True, dataset="IEMOCAPFour")[0] == names   # <= 100 clips
    with pytest.raises(AssertionError):
        MR.read_names_labels(path, "train", dataset="IEMOCAPFour")


def test_config_label_files():
    from mertools_b200 import config as C
    assert os.path.basename(C.PATH_TO_LABEL["IEMOCAPFour"]) == "label_4way.npz"
    assert os.path.basename(C.PATH_TO_LABEL["IEMOCAPSix"]) == "label_6way.npz"
    assert os.path.basename(C.PATH_TO_LABEL["MER2023"]) == "label-6way.npz"
    assert all(os.path.basename(C.PATH_TO_LABEL[d]) == "label.npz" for d in MR.SENTIMENT_CORPORA + ("MELD",))


def test_crossdim_scales_sims_by_three(config):
    """crossdim.py:77-80: SIMS / SIMSv2 valences x 3, CMU ones unchanged."""
    for ds, k in (("SIMS", 3), ("CMUMOSI", 1)):
        for dt in ("train", "test"):
            _, plain = MR.read_names_labels(config.PATH_TO_LABEL[ds], dt, dataset=ds)
            names, scaled = MR.read_crossdim_labels(config.PATH_TO_LABEL[ds], ds, dt)
            assert len(names) == len(plain)
            assert [l["val"] for l in scaled] == [l["val"] * k for l in plain]
    assert max(abs(l["val"]) for l in MR.read_crossdim_labels(config.PATH_TO_LABEL["SIMS"], "SIMS", "train")[1]) > 1


def test_crossdis_mapping_and_filtering(config, tmp_path):
    """crossdis.py:9-16,162-188: each corpus' labels onto happy / sad / neutral / angry = 0..3, the rest dropped."""
    for ds, dt in (("IEMOCAPFour", "whole"), ("MELD", "train"), ("MELD", "test")):
        raw = np.load(config.PATH_TO_LABEL[ds], allow_pickle=True)[f"{dt}_corpus"].tolist()
        names, labels = MR.read_crossdis_labels(config.PATH_TO_LABEL[ds], ds, dt)
        keep = [n for n in raw if raw[n]["emo"] in MR.CROSSDIS_MAP[ds]]
        assert names == keep
        assert [l["emo"] for l in labels] == [MR.CROSSDIS_EMO2IDX[MR.CROSSDIS_MAP[ds][raw[n]["emo"]]] for n in keep]
    # MELD: anger 0 -> angry 3, joy 1 -> happy 0, sadness 2 -> sad 1, neutral 3 -> neutral 2; 4..6 dropped
    assert [MR.CROSSDIS_EMO2IDX[MR.CROSSDIS_MAP["MELD"][e]] for e in range(4)] == [3, 0, 1, 2]
    lp, _ = S.write_merbench_corpus(str(tmp_path / "six"), "IEMOCAPSix", n=(30,), seed=5)
    raw = np.load(lp, allow_pickle=True)["whole_corpus"].tolist()
    names, labels = MR.read_crossdis_labels(lp, "IEMOCAPSix", "whole")
    assert names == [n for n in raw if raw[n]["emo"] < 4] and len(names) < 30
    os.makedirs(tmp_path / "mer")
    lp, _ = S.write_mer2023_corpus(str(tmp_path / "mer"), dim=8)
    raw = np.load(lp, allow_pickle=True)["train_corpus"].tolist()
    names, labels = MR.read_crossdis_labels(lp, "MER2023", "train")
    assert names == [n for n in raw if raw[n]["emo"] in ("neutral", "angry", "happy", "sad")]
    assert [l["emo"] for l in labels] == [MR.CROSSDIS_EMO2IDX[raw[n]["emo"]] for n in names]


def test_session_folds(config):
    """iemocap.py:78-96: fold i evaluates session i + 1 in corpus order and trains on the other four in session order."""
    names, _ = MR.read_names_labels(config.PATH_TO_LABEL["IEMOCAPFour"], "whole", dataset="IEMOCAPFour")
    folds = MR.session_split_indexes(names)
    assert len(folds) == 5
    for i, (tr, ev) in enumerate(folds):
        assert ev == [k for k, n in enumerate(names) if int(n[4]) == i + 1]
        assert tr == [k for s in range(1, 6) if s != i + 1 for k, n in enumerate(names) if int(n[4]) == s]
    with pytest.raises(AssertionError):
        MR.session_split_indexes([n for n in names if n[4] != "3"])


# ---- loaders ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(ARGV))
def test_loader_order(config, cfg):
    """Sequential train / val / test loaders for the one-fold protocols, SubsetRandomSampler over the session folds for
    IEMOCAP (train AND eval), and each split read from its own corpus."""
    args = _args(**ARGV[cfg])
    torch.manual_seed(0)
    folds, tests, trl, evl, tel = MR.load_protocol(args, config, torch.device("cpu"), say=lambda *a: None)
    tr = args.train_dataset or args.dataset
    if tr == "IEMOCAPFour":
        assert len(folds) == 5 and all(f[0] is f[1] for f in folds)
        names = folds[0][0].names
        for i in range(5):
            got = torch.cat(list(trl[i])).tolist()
            assert sorted(got) == sorted(MR.session_split_indexes(names)[i][0]) and got != sorted(got)
            assert sorted(torch.cat(list(evl[i])).tolist()) == MR.session_split_indexes(names)[i][1]
    else:
        assert len(folds) == 1 and folds[0][0] is not folds[0][1]
        state = torch.get_rng_state()
        for loader, split in ((trl[0], folds[0][0]), (evl[0], folds[0][1])):
            assert torch.cat(list(loader)).tolist() == list(range(len(split)))
        assert not torch.equal(state, torch.get_rng_state())   # each iterator draws its base seed, as the reference's
    assert len(tests) == len(tel) == (0 if args.dataset == "IEMOCAPFour" else 1)
    for ts, loader in zip(tests, tel):
        assert torch.cat(list(loader)).tolist() == list(range(len(ts)))
    if args.test_dataset is not None:
        te = args.test_dataset
        raw = np.load(config.PATH_TO_LABEL[te], allow_pickle=True)["test_corpus"].tolist()
        assert set(tests[0].names) <= set(raw) and folds[0][0].names[0] not in raw
        want = np.load(os.path.join(config.PATH_TO_FEATURES[te], "synA-UTT", tests[0].names[0] + ".npy"))
        assert np.array_equal(tests[0].a[0].numpy(), want)


# ---- metrics and names --------------------------------------------------------------------------------------------
def test_acc2_rule_against_sklearn():
    rng = np.random.default_rng(7)
    labels = np.round(rng.uniform(-3, 3, 200) * 3) / 3
    labels[::6] = 0
    preds = rng.standard_normal((200, 1)).astype(np.float32)
    res, s = FU.sentiment_calculate_results([], [], preds, labels)
    nz = labels != 0
    acc = accuracy_score(labels[nz] > 0, preds[nz, 0] > 0)
    f1 = f1_score(labels[nz] > 0, preds[nz, 0] > 0, average="weighted")
    assert res["emoacc"] == acc and res["emofscore"] == f1 and s == f"f1:{f1:.4f}_acc:{acc:.4f}"
    assert set(res) == {"valpreds", "vallabels", "emoacc", "emofscore"}
    for ds in MR.SENTIMENT_CORPORA:
        assert MR.corpus_calculate_results(ds) is FU.sentiment_calculate_results
    assert MR.corpus_calculate_results(None, "SIMS") is FU.sentiment_calculate_results
    for ds in ("MELD", "IEMOCAPFour", "IEMOCAPSix"):
        assert MR.corpus_calculate_results(ds) is FU.mer2026_calculate_results
    assert MR.corpus_calculate_results("MER2023", "MER2023") is FU.mer2026_calculate_results  # crossdis: argmax rule
    assert MR.corpus_calculate_results("MER2023") is FU.mer2023_calculate_results


def test_heads_and_names():
    assert MR.HEADS["CMUMOSI"] == (0, 1, "emo") and MR.HEADS["IEMOCAPSix"] == (6, 0, "emo")
    assert MR.HEADS["MELD"] == (7, 0, "emo") and MR.HEADS["MER2023"] == (6, 1, "emoval")
    a = _args(train_dataset="SIMS", test_dataset="CMUMOSI")
    assert MR.result_prefix(a) == ("features:synA-UTT+synT-UTT+synV-UTT_dataset:None_model:attention+utt+None"
                                   "_train:SIMS_test:CMUMOSI")
    assert MR.gain_cv_results([dict(eval_emofscore=0.5, eval_emoacc=0.25)]) == "f1:0.5000_acc:0.2500"


# ---- CPU replay of the golden runs ----------------------------------------------------------------------------------
def _replay(g, cfg, config):
    """The mirror's host logic (label readers, protocol loaders, initial weights, result names) driving the oracle's
    fp32 CPU forward and torch.optim.Adam as the unmodified script ran (dropout 0, loss = CE when output_dim1 != 0 plus
    MSE when output_dim2 != 0)."""
    torch.manual_seed(int(g["seed"]))
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    args = _args(**ARGV[cfg])
    cross = args.train_dataset is not None
    if cross:
        o1, o2, _ = (0, 1, "emo") if args.train_dataset in MR.SENTIMENT_CORPORA else (4, 0, "emo")
    else:
        o1, o2, _ = MR.HEADS[args.dataset]
    args.output_dim1, args.output_dim2 = o1, o2
    prefix = MR.result_prefix(args)
    folds, tests, trl, evl, tel = MR.load_protocol(args, config, torch.device("cpu"), say=lambda *a: None)
    calc = MR.corpus_calculate_results(args.dataset, args.train_dataset)
    dims = folds[0][0].dims
    E, F = int(g["epochs"]), len(folds)
    out = dict(train=np.zeros((F, E)), eval=np.zeros((F, E)), test=np.zeros((len(tests), F, E)), best=[],
               enames=[], tnames=[], save=[])

    def loss_of(eo, vo, emo, val):
        ce = OF.losses(eo, torch.zeros(len(eo), 0), emo, torch.zeros(len(eo), 0))[0] if o1 else 0.0
        mse = OF.losses(torch.zeros(len(vo), 1), vo, torch.zeros(len(vo), dtype=torch.long), val)[1] if o2 else 0.0
        return ce + mse

    def evaluate(sd, split, loader):
        losses, eo_all, vo_all, order = [], [], [], []
        with torch.no_grad():
            for b in loader:
                _, eo, vo = OF.attention_forward(sd, split.a[b], split.t[b], split.v[b])
                losses.append(float(loss_of(eo, vo, split.emo[b], split.val[b])))
                eo_all.append(eo.numpy())
                vo_all.append(vo.numpy())
                order += b.tolist()
        eo, vo = np.concatenate(eo_all), np.concatenate(vo_all)
        res, _ = calc(eo if o1 else [], split.emo[order].numpy() if o1 else [], vo if o2 else [],
                      split.val[order].numpy() if o2 else [])
        return dict(loss=np.mean(losses), names=[split.names[i] for i in order], eo=eo, vo=vo, **res)

    for f in range(F):
        sd = {k: v.clone().requires_grad_(True)
              for k, v in FU.reference_init(args.feat_type, *dims, 64, o1, o2).items()}
        opt = torch.optim.Adam(list(sd.values()), lr=1e-3, weight_decay=1e-5)
        metrics, store = [], []
        for ep in range(E):
            losses, order = [], []
            tr = folds[f][0]
            for b in trl[f]:
                opt.zero_grad()
                _, eo, vo = OF.attention_forward(sd, tr.a[b], tr.t[b], tr.v[b])
                loss = loss_of(eo, vo, tr.emo[b], tr.val[b])
                loss.backward()
                opt.step()
                losses.append(float(loss))
                order += b.tolist()
            out["train"][f, ep] = np.mean(losses)
            ev = evaluate(sd, folds[f][1], evl[f])
            out["eval"][f, ep] = ev["loss"]
            ts = [evaluate(sd, t, tel[j]) for j, t in enumerate(tests)]
            for j, t in enumerate(ts):
                out["test"][j, f, ep] = t["loss"]
            metrics.append(ev["emofscore"])
            store.append(dict(eval_emofscore=ev["emofscore"], eval_emoacc=ev["emoacc"], tests=ts))
            if ep == 0:
                out["enames"].append(ev["names"])
                out["tnames"].append([tr.names[i] for i in order])
        out["best"].append(int(np.argmax(metrics)))
        out["save"].append(store[out["best"][-1]])
    saved = [f"cv_{prefix}_{MR.gain_cv_results(out['save'])}"]
    for j in range(len(tests)):
        eo = np.mean([s["tests"][j]["eo"] for s in out["save"]], axis=0)
        vo = np.mean([s["tests"][j]["vo"] for s in out["save"]], axis=0)
        _, r = calc(eo if o1 else [], tests[j].emo.numpy() if o1 else [], vo if o2 else [],
                    tests[j].val.numpy() if o2 else [])
        saved.append(f"test{j + 1}_{prefix}_{r}")
    out["saved"] = saved
    out["dims"] = list(dims)
    return out


@pytest.mark.parametrize("cfg", list(ARGV))
def test_cpu_replay_of_the_golden(config, cfg):
    g = np.load(GOLDEN)
    pre = f"{cfg}_"
    r = _replay(g, cfg, config)
    assert r["dims"] == list(g[pre + "feat_dims"])
    assert len(r["best"]) == int(g[pre + "folds"])
    for f in range(len(r["best"])):
        assert r["enames"][f] == list(g[f"{pre}fold{f}_eval_names_epoch0"]), f"fold {f}: eval split / order"
        assert r["tnames"][f] == list(g[f"{pre}fold{f}_train_names_epoch0"]), f"fold {f}: train order"
    assert r["best"] == list(g[pre + "best_index"])
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()  # noqa: E731
    assert rel(r["train"], g[pre + "train_loss"]) < 1e-5
    assert rel(r["eval"], g[pre + "eval_loss"]) < 1e-5
    if r["test"].size:
        assert rel(r["test"], g[pre + "test_loss"]) < 1e-5
    assert r["saved"] == list(g[pre + "saved"])
