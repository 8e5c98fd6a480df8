"""MER2023 baseline training CLI -- the H100 mirror of MER2023/main-release.py, the trainer MER2023/run_release.sh
runs after feature extraction: ``--model_type mlp | attention`` over a free ``--layers`` list, five-fold
cross-validation on train, every test set evaluated every epoch, and the fold-averaged predictions written as the
challenge's ``{set}-pred-{time}.csv`` submission files.

Same flags (:533-560), same feature reader (func_read_one, :49-72: ``feature_root/name*`` must match exactly one
``.npy`` file or per-face directory), same label file (``label-6way.npz`` ``{split}_corpus``, :74-117), same folds
(:157-181, python ``random``), same loaders (SubsetRandomSampler for train and eval, test sets in order), same
per-epoch protocol and best-epoch rule (f1 - 0.25 mse, first best, :625-658) and same outputs (:661-703).  As in the
reference, ``--dropout`` is parsed and ignored: the nets train with dropout 0.3 (:601-612).

What changes is where the work happens: the features are read once and live on the GPU, torch's own ``DataLoader`` /
``SubsetRandomSampler`` only shuffle sample indices, batches are index-selected on the device, and every training step
is one MlpFusionNet.train_step (csrc/fusion_mlp.cu).  The reference uses one GPU and so does this trainer: under
torchrun with more than one process it refuses to start.
"""
from __future__ import annotations

import argparse
import glob
import os
import random
import time

import numpy as np
import torch

from . import shard
from .fusion_mlp import REFERENCE_DROPOUT, MlpFusionNet, check_batch, reference_init
from .main_release import get_loaders, random_split_indexes

EMOS = ["neutral", "angry", "happy", "sad", "worried", "surprise"]      # main-release.py:41
EMO2IDX = {e: i for i, e in enumerate(EMOS)}
IDX2EMO = dict(enumerate(EMOS))
DATASETS = ("MER2023",)   # what the reference's config.py knows


# ---- data ------------------------------------------------------------------------------------------------------------
def func_read_one(feature_root, name):
    """main-release.py:49-72: the one entry ``feature_root/name*`` -> a squeezed ``.npy``, or a directory's per-face
    ``.npy`` files stacked in sorted order, squeezed and (when 2-D) averaged over the faces."""
    matches = glob.glob(os.path.join(feature_root, name + "*"))
    assert len(matches) == 1, f"{feature_root}/{name}* matches {len(matches)} entries, not exactly one"
    path = matches[0]
    if path.endswith(".npy"):
        feature = [np.load(path).squeeze()]
    else:
        feature = [np.load(os.path.join(path, f)) for f in sorted(os.listdir(path))]
    feat = np.array(feature).squeeze()
    if len(feat) == 0:
        print("feature has errors!!")
    elif feat.ndim == 2:
        feat = np.mean(feat, axis=0)
    return feat


def read_names_labels(label_path, data_type, debug=False):
    """main-release.py:74-98 (task 'whole'): names in corpus order, labels {'emo': index, 'val': valence}."""
    assert data_type in ("train", "test1", "test2", "test3"), data_type
    corpus = np.load(label_path, allow_pickle=True)[f"{data_type}_corpus"].tolist()
    names = list(corpus)
    labels = [{"emo": EMO2IDX[corpus[n]["emo"]], "val": corpus[n]["val"]} for n in names]
    if debug:
        names, labels = names[:100], labels[:100]
    return names, labels


class Split:
    """One MERDataset (:123-146) resident on the device: A / T / V [N, D] fp32, emo int64, val fp32."""

    def __init__(self, label_path, roots, data_type, device, debug=False):
        self.names, labels = read_names_labels(label_path, data_type, debug)
        feats = []
        for root in roots:
            rows = [func_read_one(root, n) for n in self.names]
            feats.append(np.array(rows).astype(np.float32))
            print(f"Input feature {root} ===> dim is {feats[-1].shape[-1]}")
        self.a, self.t, self.v = (torch.from_numpy(f).to(device) for f in feats)
        self.dims = tuple(int(f.shape[-1]) for f in feats)
        self.emo = torch.tensor([l["emo"] for l in labels], dtype=torch.int64, device=device)
        self.val = torch.tensor([float(l["val"]) for l in labels], dtype=torch.float32, device=device)

    def __len__(self):
        return len(self.names)


# ---- metrics and outputs (main-release.py:403-527) ---------------------------------------------------------------------
def overall_metric(emo_fscore, val_mse):
    return emo_fscore - val_mse * 0.25


def average_folder_results(folder_save, testname):
    """:407-432: per name, the mean over the folds of the emotion logits (argmax -> 'emo') and of the valence."""
    name2preds = {}
    for fold in folder_save:
        for name, emoprob, valpred in zip(fold[f"{testname}_names"], fold[f"{testname}_emoprobs"],
                                          fold[f"{testname}_valpreds"]):
            name2preds.setdefault(name, []).append({"emo": emoprob, "val": valpred})
    out = {}
    for name, preds in name2preds.items():
        avg_emoprob = np.mean([p["emo"] for p in preds], axis=0)
        out[name] = {"emo": np.argmax(avg_emoprob), "val": np.mean([p["val"] for p in preds]),
                     "emoprob": avg_emoprob}
    return out


def gain_name2feat(folder_save, testname):
    """:434-443: fold 0's features of every test clip."""
    assert len(folder_save) >= 1
    return dict(zip(folder_save[0][f"{testname}_names"], folder_save[0][f"{testname}_embeddings"]))


def write_to_csv_pred(name2preds, save_path):
    """:445-455: columns name, discrete, valence (np.column_stack makes every column a string, as there)."""
    import pandas as pd
    names = list(name2preds)
    emos = [IDX2EMO[name2preds[n]["emo"]] for n in names]
    vals = [name2preds[n]["val"] for n in names]
    pd.DataFrame(data=np.column_stack([names, emos, vals]), columns=["name", "discrete", "valence"]).to_csv(
        save_path, index=False)


def _read_csv(path, with_val):
    import pandas as pd
    out = {}
    for _, row in pd.read_csv(path).iterrows():
        out[row["name"]] = {"emo": EMO2IDX[row["discrete"]], **({"val": row["valence"]} if with_val else {})}
    return out


def report_results_on_test1_test2(test_label, test_pred):
    """:457-494: weighted F1, valence MSE and the overall metric over every labelled clip."""
    from sklearn.metrics import f1_score, mean_squared_error
    name2label, name2pred = _read_csv(test_label, True), _read_csv(test_pred, True)
    print(f"labeled samples: {len(name2label)}")
    print(f"predict samples: {len(name2pred)}")
    assert len(name2pred) == len(name2label), "make sure len(name2pred)=len(name2label)"
    names = list(name2label)
    emo_fscore = f1_score([name2label[n]["emo"] for n in names], [name2pred[n]["emo"] for n in names],
                          average="weighted")
    val_mse = mean_squared_error([name2label[n]["val"] for n in names], [name2pred[n]["val"] for n in names])
    final_metric = overall_metric(emo_fscore, val_mse)
    print(f"emo results (weighted f1 score): {emo_fscore:.4f}")
    print(f"val results (mse): {val_mse:.4f}")
    print(f"overall metric: {final_metric:.4f}")
    return emo_fscore, val_mse, final_metric


def report_results_on_test3(test_label, test_pred):
    """:498-527: weighted F1 over the labelled clips only (test3 labels a subset); -100 for the other two."""
    from sklearn.metrics import f1_score
    name2label, name2pred = _read_csv(test_label, False), _read_csv(test_pred, False)
    print(f"labeled samples: {len(name2label)}")
    print(f"predict samples: {len(name2pred)}")
    assert len(name2pred) >= len(name2label)
    names = list(name2label)
    emo_fscore = f1_score([name2label[n]["emo"] for n in names], [name2pred[n]["emo"] for n in names],
                          average="weighted")
    print(f"emo results (weighted f1 score): {emo_fscore:.4f}")
    return emo_fscore, -100, -100


def save_root_suffix(save_root, audio_feature, text_feature, video_feature):
    """:572-578: -unimodal / -bimodal / -trimodal by the number of distinct feature names."""
    n = len({audio_feature, text_feature, video_feature})
    return f"{save_root}-" + {1: "unimodal", 2: "bimodal", 3: "trimodal"}[n]


# ---- one pass over a split (main-release.py:321-397) -------------------------------------------------------------------
def run_pass(args, net, split, batches, train=False, lr=None, l2=None, masks=None):
    """``batches``: index tensors in the reference's loader order.  Training: one step per batch (``masks(i)`` gives
    batch i's keep-masks when replaying recorded ones); evaluation: the eval forward.  Returns the reference's
    save_results dict plus 'loss' (the train batches' mean CE + MSE; None when not training)."""
    from sklearn.metrics import accuracy_score, f1_score, mean_squared_error
    dev = split.emo.device
    names, emo_probs, val_preds, embeddings, losses, order = [], [], [], [], [], []
    for i, b in enumerate(batches):
        b = b.to(dev)
        names += [split.names[j] for j in b.tolist()]
        order.append(b)
        a, t, v = (x.index_select(0, b) for x in (split.a, split.t, split.v))
        check_batch(args.model_type, len(b))
        if train:
            loss3, feats, eo, vo = net.train_step(a, t, v, split.emo.index_select(0, b), split.val.index_select(0, b),
                                                  lr=lr, weight_decay=l2,
                                                  ext_masks=None if masks is None else masks(i))
            losses.append(loss3[2:3].clone())
        else:
            feats, eo, vo = net(a, t, v)
        emo_probs.append(eo.clone())
        val_preds.append(vo.clone())
        embeddings.append(feats.clone())
    order = torch.cat(order)
    emo_probs = torch.cat(emo_probs).cpu().numpy()
    val_preds = torch.cat(val_preds).cpu().numpy()
    emo_labels = split.emo.index_select(0, order).cpu().numpy()
    val_labels = split.val.index_select(0, order).cpu().numpy()
    emo_preds = np.argmax(emo_probs, 1)
    res = dict(val_mse=mean_squared_error(val_labels, val_preds),
               emo_fscore=f1_score(emo_labels, emo_preds, average="weighted"),
               emo_accuracy=accuracy_score(emo_labels, emo_preds), emo_probs=emo_probs, val_preds=val_preds,
               emo_labels=emo_labels, val_labels=val_labels, names=names,
               loss=float(torch.cat(losses).mean()) if losses else None)
    if args.savewhole:
        res["embeddings"] = torch.cat(embeddings).cpu().numpy()
    return res


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--dataset", type=str, default=None)
    p.add_argument("--train_dataset", type=str, default=None)
    p.add_argument("--test_dataset", type=str, default=None)
    p.add_argument("--audio_feature", type=str, default=None)
    p.add_argument("--text_feature", type=str, default=None)
    p.add_argument("--video_feature", type=str, default=None)
    p.add_argument("--debug", action="store_true", default=False)
    p.add_argument("--test_sets", type=str, default="test1,test2")
    p.add_argument("--save_root", type=str, default="./saved")
    p.add_argument("--savewhole", action="store_true", default=False)
    p.add_argument("--layers", type=str, default="256,128")
    p.add_argument("--n_classes", type=int, default=-1)
    p.add_argument("--num_folder", type=int, default=-1)
    p.add_argument("--model_type", type=str, default="mlp")
    p.add_argument("--lr", type=float, default=0.0001)
    p.add_argument("--l2", type=float, default=0.00001)
    p.add_argument("--dropout", type=float, default=0.5)   # parsed and unused, as in the reference
    p.add_argument("--batch_size", type=int, default=32)
    p.add_argument("--num_workers", type=int, default=0)
    p.add_argument("--epochs", type=int, default=100)
    p.add_argument("--seed", type=int, default=100)        # parsed and unused, as in the reference
    p.add_argument("--gpu", default=0, type=int)
    return p


def _batches(loader):
    return [torch.as_tensor(b) for b in loader]


def _chunks(order, bs):
    order = torch.as_tensor(np.asarray(order, dtype=np.int64))
    return [order[i:i + bs] for i in range(0, len(order), bs)]


def main(args, config=None, replay=None, make_net=None, device=None):
    """Runs the protocol of main-release.py:561-703 and returns the paths it wrote.

    For deterministic replays of a recorded reference run (tests, the float64 studies): ``replay`` may supply
    ``init_rng(fold)`` (torch's CPU generator state before fold ``fold`` builds its model), ``order(fold, epoch,
    which)`` (the sample order of the 'train' / 'eval' sampler) and ``masks(fold, epoch, batch)`` (that training
    batch's dropout keep-masks); ``make_net(kind, dims, state_dict)`` replaces the device net (the oracle's, on the
    CPU) and ``device`` the GPU."""
    if config is None:
        from . import config as config  # noqa: PLW0127
    rank, world = shard.env_rank_world()
    if world > 1:
        raise SystemExit("main_release_mer2023 trains on one GPU, as MER2023/main-release.py does: run it without "
                         "torchrun (or with --nproc-per-node 1)")
    args.n_classes = 6
    args.num_folder = 5
    args.test_sets = args.test_sets.split(",") if isinstance(args.test_sets, str) else list(args.test_sets)
    if args.dataset is not None:
        args.train_dataset = args.test_dataset = args.dataset
    assert args.train_dataset is not None and args.test_dataset is not None, "--dataset (or --train_dataset and " \
        "--test_dataset) is required"
    for ds in (args.train_dataset, args.test_dataset):
        assert ds in DATASETS, f"MER2023/main-release.py reads MER2023-format corpora only ({DATASETS}), not {ds}"
    assert args.model_type in ("mlp", "attention"), f"--model_type mlp | attention, not {args.model_type}"
    args.save_root = save_root_suffix(args.save_root, args.audio_feature, args.text_feature, args.video_feature)
    if device is None:
        torch.cuda.set_device(args.gpu)
        device = torch.device("cuda", args.gpu)
    print(args)

    print("====== Reading Data =======")
    froot = lambda ds: [os.path.join(config.PATH_TO_FEATURES[ds], f)  # noqa: E731
                        for f in (args.audio_feature, args.text_feature, args.video_feature)]
    train = Split(config.PATH_TO_LABEL[args.train_dataset], froot(args.train_dataset), "train", device, args.debug)
    folds = random_split_indexes(len(train), args.num_folder)
    tests = [Split(config.PATH_TO_LABEL[args.test_dataset], froot(args.test_dataset), ts, device, args.debug)
             for ts in args.test_sets]
    train_loaders, eval_loaders, test_loaders = get_loaders(len(train), folds, [len(t) for t in tests],
                                                            args.batch_size, args.num_workers)
    adim, tdim, vdim = train.dims
    print(f"audio dimension: {adim}; text dimension: {tdim}; video dimension: {vdim}")

    print("====== Training and Evaluation =======")
    folder_save, folder_evalres = [], []
    name_time = time.time()
    for ii in range(args.num_folder):
        print(f">>>>> Cross-validation: training on the {ii + 1} folder >>>>>")
        start_time = name_time = time.time()
        if replay is not None:
            torch.set_rng_state(replay.init_rng(ii))
        sd = reference_init(args.model_type, adim, tdim, vdim, args.layers, args.n_classes, 1)
        if make_net is not None:
            net = make_net(args.model_type, (adim, tdim, vdim), sd)
        else:
            net = MlpFusionNet(args.model_type, adim, tdim, vdim, args.layers, args.n_classes, 1,
                               dropout=REFERENCE_DROPOUT, device=device, max_batch=max(args.batch_size, 2),
                               seed=random.randint(0, 2 ** 31 - 1) if replay is None else 0).load_state_dict(sd)
        eval_metrics, eval_fscores, eval_valmses, test_save = [], [], [], []
        for epoch in range(args.epochs):
            if replay is None:
                tr_b, ev_b = _batches(train_loaders[ii]), _batches(eval_loaders[ii])
                masks = None
            else:
                tr_b = _chunks(replay.order(ii, epoch, "train"), args.batch_size)
                ev_b = _chunks(replay.order(ii, epoch, "eval"), args.batch_size)
                masks = lambda i, ii=ii, epoch=epoch: replay.masks(ii, epoch, i)  # noqa: E731
            train_res = run_pass(args, net, train, tr_b, True, args.lr, args.l2, masks)
            eval_res = run_pass(args, net, train, ev_b)
            eval_metric = overall_metric(eval_res["emo_fscore"], eval_res["val_mse"])
            eval_metrics.append(eval_metric)
            eval_fscores.append(eval_res["emo_fscore"])
            eval_valmses.append(eval_res["val_mse"])
            store = {"eval_emoprobs": eval_res["emo_probs"], "eval_valpreds": eval_res["val_preds"],
                     "eval_names": eval_res["names"], "train_loss": train_res["loss"],
                     "train_fscore": train_res["emo_fscore"], "train_valmse": train_res["val_mse"],
                     "eval_fscore": eval_res["emo_fscore"], "eval_valmse": eval_res["val_mse"],
                     "train_names": train_res["names"]}
            print("epoch:%d; train_fscore:%.4f; eval_metric:%.4f" % (epoch + 1, train_res["emo_fscore"], eval_metric))
            for jj, test_loader in enumerate(test_loaders):
                ts = args.test_sets[jj]
                res = run_pass(args, net, tests[jj], _batches(test_loader))
                store[f"{ts}_emoprobs"], store[f"{ts}_valpreds"] = res["emo_probs"], res["val_preds"]
                store[f"{ts}_names"] = res["names"]
                store[f"{ts}_fscore"], store[f"{ts}_valmse"] = res["emo_fscore"], res["val_mse"]
                if args.savewhole:
                    store[f"{ts}_embeddings"] = res["embeddings"]
            test_save.append(store)
        print(f"Step3: saving and testing on the {ii + 1} folder")
        best_index = int(np.argmax(np.array(eval_metrics)))
        folder_save.append(test_save[best_index])
        folder_evalres.append([eval_fscores[best_index], eval_valmses[best_index]])
        print(f">>>>> Finish: training on the {ii + 1} folder, best epoch: {best_index + 1}, "
              f"duration: {time.time() - start_time} >>>>>")
        if replay is not None and hasattr(replay, "on_fold"):
            replay.on_fold(ii, test_save, best_index, net)
        del net

    print("====== Gain predition on test data =======")
    save_modelroot = os.path.join(args.save_root, "model")
    save_predroot = os.path.join(args.save_root, "prediction")
    os.makedirs(save_predroot, exist_ok=True)
    os.makedirs(save_modelroot, exist_ok=True)
    feature_name = f"{args.audio_feature}+{args.text_feature}+{args.video_feature}"
    cv_fscore, cv_valmse = np.mean(np.array(folder_evalres), axis=0)
    cv_metric = overall_metric(cv_fscore, cv_valmse)
    res_name = f"f1:{cv_fscore:.4f}_val:{cv_valmse:.4f}_metric:{cv_metric:.4f}"
    save_path = f"{save_modelroot}/cv_features:{feature_name}_{res_name}_{name_time}.npz"
    print(f"save results in {save_path}")
    np.savez_compressed(save_path, args=np.array(args, dtype=object))
    written = [save_path]
    for setname in args.test_sets:
        pred_path = f"{save_predroot}/{setname}-pred-{name_time}.csv"
        label_path = f"./dataset-release/{setname}-label.csv"
        name2preds = average_folder_results(folder_save, setname)
        write_to_csv_pred(name2preds, pred_path)
        written.append(pred_path)
        res_name = "nores"
        if os.path.exists(label_path):
            if setname in ("test1", "test2"):
                emo_fscore, val_mse, final_metric = report_results_on_test1_test2(label_path, pred_path)
            if setname == "test3":
                emo_fscore, val_mse, final_metric = report_results_on_test3(label_path, pred_path)
            res_name = f"f1:{emo_fscore:.4f}_val:{val_mse:.4f}_metric:{final_metric:.4f}"
        save_path = f"{save_modelroot}/{setname}_features:{feature_name}_{res_name}_{name_time}.npz"
        print(f"save results in {save_path}")
        extra = dict(name2feats=gain_name2feat(folder_save, setname)) if args.savewhole else {}
        np.savez_compressed(save_path, name2preds=name2preds, **extra, args=np.array(args, dtype=object))
        written.append(save_path)
    return written, folder_save, name_time


if __name__ == "__main__":
    main(build_parser().parse_args())
