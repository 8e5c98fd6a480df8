"""Attention-fusion training CLI — H100 mirror of MERBench/main-release.py for
``--model attention --feat_type utt --dataset MER2023`` (the configuration of SURVEY.md §8 rows
a9-a12).  Same flags (:93-124), same hyper-parameter handling (model-tune.yaml ``attention`` grid or
``--hyper_path``, :159-165), same label / feature file formats (toolkit/dataloader/mer2023.py:82-104,
toolkit/utils/read_data.py:15-41,92-97), same 5-fold protocol (mer2023.py:108-134), metrics
(toolkit/utils/metric.py) and result files ``cv_*.npz`` / ``test{j}_*.npz`` (:256-272).

What changes is where the work happens: all features live on the GPU once, torch's own ``DataLoader`` /
``SubsetRandomSampler`` only shuffle and batch sample INDICES (so the order of samples and the consumption of
torch's generator are the reference's by construction), batches are index-selected on the device, and every
training step is one fused FusionNet.train_step (forward + CE/MSE + backward + Adam in two kernels).  The golden of
the unmodified script (tests/golden/make_golden_main_release.py) is reproduced fold for fold, epoch for epoch.

Under ``python -m torch.distributed.run --nproc-per-node W -m mertools_b200.main_release ...`` the trainer is
data-parallel (SURVEY.md §8e): rank 0's seed and initial weights are broadcast once, every rank draws the same
permutation, takes the rank-strided slice ``batch[rank::W]`` of each reference batch, and the flat gradient (with
the loss scalars) is all-reduced once per step; every rank evaluates the full splits, rank 0 writes the result files.
"""
from __future__ import annotations

import argparse
import os
import random
import time

import numpy as np
import torch

from . import shard
from .fusion import Adam, get_models, mer2023_calculate_results

EMOS_MER = ["neutral", "angry", "happy", "sad", "worried", "surprise"]      # toolkit/globals.py:2
EMO2IDX = {e: i for i, e in enumerate(EMOS_MER)}
ATTENTION_GRID = dict(hidden_dim=[64, 128, 256], dropout=[0.2, 0.3, 0.4, 0.5], grad_clip=[-1.0],
                      lr=[1e-3, 1e-4])                                       # toolkit/model-tune.yaml:76-80


# ---- data (host side, same file formats as the reference) ---------------------------------------
def read_names_labels(label_path, data_type, debug=False):
    """mer2023.py:82-104."""
    assert data_type in ("train", "test1", "test2", "test3")
    corpus = np.load(label_path, allow_pickle=True)[f"{data_type}_corpus"].tolist()
    names, labels = [], []
    for name, label in corpus.items():
        names.append(name)
        val = label["val"] if ("val" in label and label["val"] != "") else -10
        labels.append({"emo": EMO2IDX[label["emo"]], "val": val})
    if debug:
        names, labels = names[:100], labels[:100]
    return names, labels


def read_utt_feature(feature_root, name):
    """read_data.py:15-41 + align_to_utt (:92-97): one clip -> [D] (mean over time when 2-D)."""
    path = os.path.join(feature_root, name + ".npy")
    d = os.path.join(feature_root, name)
    if os.path.exists(path):
        feat = np.load(path).squeeze()
    elif os.path.isdir(d):
        feat = np.array([np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))]).squeeze()
    else:
        raise Exception("feature path or dir do not exist!")
    if feat.ndim == 1:
        feat = feat[np.newaxis, :]
    return np.mean(feat, axis=0)


def read_frm_feature(feature_root, name):
    """read_data.py:15-41 (func_read_one_feat): one clip -> [T, D] (a single vector becomes [1, D])."""
    path = os.path.join(feature_root, name + ".npy")
    d = os.path.join(feature_root, name)
    if os.path.exists(path):
        feat = np.load(path).squeeze()
    elif os.path.isdir(d):
        feat = np.array([np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))]).squeeze()
    else:
        raise Exception("feature path or dir do not exist!")
    if feat.ndim == 1:
        feat = feat[np.newaxis, :]
    return feat


def random_split_indexes(whole_num, num_folder):
    """mer2023.py:108-134 (python ``random`` shuffle, last fold takes the remainder)."""
    indices = np.arange(whole_num)
    random.shuffle(indices)
    each = int(whole_num / num_folder)
    folds = [indices[each * i: each * (i + 1)] for i in range(num_folder - 1)] + [indices[each * (num_folder - 1):]]
    out = []
    for i in range(num_folder):
        train = [x for j in range(num_folder) if j != i for x in folds[j]]
        out.append([train, list(folds[i])])
    return out


class DeviceSplit:
    """One corpus split resident on the GPU: A/T/V fp32 -- [N, D] for feat_type 'utt', [N, T_m, D] for the
    frame-level types (shaped exactly as Data_Feat does, feat_data.py:33-44) -- emo int64, val fp32."""

    def __init__(self, args, names, labels, config, device):
        root = config.PATH_TO_FEATURES[args.dataset]
        feats = []
        if args.feat_type == "utt":
            for fname in (args.audio_feature, args.text_feature, args.video_feature):
                fr = os.path.join(root, fname)
                feats.append(np.stack([read_utt_feature(fr, n) for n in names]).astype(np.float32))
        else:
            from . import frame_features as FF
            raw = [[read_frm_feature(os.path.join(root, fname), n) for n in names]
                   for fname in (args.audio_feature, args.text_feature, args.video_feature)]
            shaped = FF.shape_split(raw[0], raw[1], raw[2], args.feat_type, args.feat_scale)
            feats = [np.array(x).astype(np.float32) for x in shaped]  # torch.FloatTensor(np.array(...)) in the collater
        self.names = names
        self.a, self.t, self.v = (torch.from_numpy(f).to(device) for f in feats)
        self.emo = torch.tensor([l["emo"] for l in labels], dtype=torch.int64, device=device)
        self.val = torch.tensor([l["val"] for l in labels], dtype=torch.float32, device=device).view(-1, 1)
        self.dims = tuple(int(f.shape[-1]) for f in feats)

    def __len__(self):
        return len(self.names)


class _Indices(torch.utils.data.Dataset):
    """What the DataLoaders iterate: sample numbers.  The features never leave the GPU."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return int(i)


def get_loaders(n_train, folds, n_tests, batch_size, num_workers=0):
    """The loader objects of MER2023.get_loaders (mer2023.py:31-79), over sample indices: SubsetRandomSampler for the
    train AND the eval part of each fold (the reference shuffles both), sequential order for the test sets."""
    from torch.utils.data import DataLoader
    from torch.utils.data.sampler import SubsetRandomSampler
    train_set = _Indices(n_train)
    mk = lambda idxs: DataLoader(train_set, batch_size=batch_size, sampler=SubsetRandomSampler(idxs),  # noqa: E731
                                 num_workers=num_workers)
    train_loaders = [mk(tr) for tr, _ in folds]
    eval_loaders = [mk(ev) for _, ev in folds]
    test_loaders = [DataLoader(_Indices(n), batch_size=batch_size, num_workers=num_workers, shuffle=False)
                    for n in n_tests]
    return train_loaders, eval_loaders, test_loaders


calculate_results = mer2023_calculate_results  # mer2023.py:137-155


def gain_metric_from_results(res, metric_name="emoval"):
    """toolkit/utils/metric.py:15-32."""
    if metric_name == "emoval":
        return res["emofscore"] - 0.25 * res["valmse"]
    if metric_name == "emo":
        return res["emofscore"]
    if metric_name == "val":
        return -res["valmse"]
    return -res["loss"]


def _gather_strided(local, n_global, rank, world):
    """Rows ``rank::world`` of a data-parallel batch from every rank -> the [n_global, C] batch in its own order."""
    import torch.distributed as dist
    per = -(-n_global // world)
    pad = torch.zeros(per, local.shape[1], dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    out = torch.empty(n_global, local.shape[1], dtype=local.dtype, device=local.device)
    for r in range(world):
        out[r::world] = parts[r][:len(range(r, n_global, world))]
    return out


# ---- one pass over a split (main-release.py:17-87) ------------------------------------------------
def run_split(args, net, split, loader, optimizer=None, train=False, rank=0, world_size=1):
    """``loader`` yields batches of sample indices in the reference's order.  Training: one fused step per batch
    (under data parallelism on rows ``rank::world_size`` of it); evaluation: eval forward + the two losses."""
    dev = split.a.device
    names, emo_probs, val_preds, losses, order = [], [], [], [], []
    net.train(train)
    for b in loader:
        names += [split.names[i] for i in b.tolist()]
        b = b.to(dev)
        order.append(b)
        mine = b[rank::world_size] if (train and world_size > 1) else b
        a, t, v = split.a.index_select(0, mine), split.t.index_select(0, mine), split.v.index_select(0, mine)
        emo, val = split.emo.index_select(0, mine), split.val.index_select(0, mine)
        if train:
            loss3, eo, vo = net.train_step(a, t, v, emo, val, lr=optimizer.lr, betas=optimizer.betas,
                                           eps=optimizer.eps, weight_decay=optimizer.weight_decay,
                                           world_size=world_size, global_batch=len(b))
            losses.append(loss3[2:3].clone())
            if world_size > 1:
                eo, vo = (_gather_strided(x, len(b), rank, world_size) for x in (eo, vo))
        else:
            _, eo, vo, _ = net({"audios": a, "texts": t, "videos": v})
            ce = torch.nn.functional.cross_entropy(eo, emo, reduction="sum") / len(eo)
            mse = torch.nn.functional.mse_loss(vo, val, reduction="sum") / len(vo)
            losses.append((ce + mse).view(1))
        emo_probs.append(eo.clone())
        val_preds.append(vo.clone())
    order = torch.cat(order)
    emo_probs = torch.cat(emo_probs).cpu().numpy()
    val_preds = torch.cat(val_preds).cpu().numpy()
    emo_labels = split.emo.index_select(0, order).cpu().numpy()
    val_labels = split.val.index_select(0, order).cpu().numpy()
    res, _ = calculate_results(emo_probs, emo_labels, val_preds, val_labels)
    return dict(names=names, loss=np.mean(torch.cat(losses).cpu().numpy()), **res)


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--dataset", type=str, default="MER2023")
    p.add_argument("--save_root", type=str, default="./saved")
    p.add_argument("--debug", action="store_true", default=False)
    p.add_argument("--audio_feature", type=str, default=None)
    p.add_argument("--text_feature", type=str, default=None)
    p.add_argument("--video_feature", type=str, default=None)
    p.add_argument("--feat_type", type=str, default="utt")
    p.add_argument("--feat_scale", type=int, default=None)
    p.add_argument("--e2e_name", type=str, default=None)
    p.add_argument("--hyper_path", type=str, default=None)
    p.add_argument("--model", type=str, default="attention")
    p.add_argument("--lr", type=float, default=None)
    p.add_argument("--l2", type=float, default=0.00001)
    p.add_argument("--batch_size", type=int, default=32)
    p.add_argument("--num_workers", type=int, default=0)
    p.add_argument("--epochs", type=int, default=100)
    p.add_argument("--print_iters", type=int, default=1e8)
    p.add_argument("--gpu", default=0, type=int)
    return p


def _init_distributed(args):
    """torchrun environment -> (rank, world).  One process per GPU; LOCAL_RANK overrides --gpu."""
    rank, world = shard.env_rank_world()
    if world > 1:
        import torch.distributed as dist
        args.gpu = int(os.environ.get("LOCAL_RANK", rank))
        torch.cuda.set_device(args.gpu)
        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=torch.device("cuda", args.gpu))
        # the reference seeds nothing: make every rank continue rank 0's random streams
        seed = torch.tensor([random.randrange(2 ** 31) if rank == 0 else 0], dtype=torch.int64, device="cuda")
        dist.broadcast(seed, 0)
        random.seed(int(seed))
        torch.manual_seed(int(seed))
    return rank, world


def main(args, config=None, log=None):
    """``log`` (optional dict) receives per-fold, per-epoch train / eval / test losses and the fold membership --
    what tests/golden/main_release_golden.npz holds for the unmodified script."""
    if config is None:
        from . import config as config  # noqa: PLW0127
    assert args.model == "attention" and args.dataset == "MER2023", \
        "the H100 path covers --model attention --dataset MER2023 (SURVEY.md §8)"
    rank, world = _init_distributed(args)
    torch.cuda.set_device(args.gpu)
    device = torch.device("cuda", args.gpu)
    say = print if rank == 0 else (lambda *a, **k: None)
    # pre-compression of the frame-level types (main-release.py:131-142)
    if args.feat_type == "utt":
        args.feat_scale = 1
    else:
        assert args.feat_type in ("frm_align", "frm_unalign"), args.feat_type
        for f in (args.audio_feature, args.text_feature, args.video_feature):
            assert f.endswith("FRA"), f"feat_type {args.feat_type} needs frame-level features, got {f}"
        args.feat_scale = 6 if args.feat_type == "frm_align" else 12
    feats = [f for f in (args.audio_feature, args.text_feature, args.video_feature) if f is not None]
    args.save_root = f"{args.save_root}-" + {0: "others", 1: "unimodal", 2: "bimodal", 3: "trimodal"}[len(set(feats))]
    if args.hyper_path is None:
        cfg = {k: v[random.randint(0, len(v) - 1)] for k, v in ATTENTION_GRID.items()}   # func_random_select
    else:
        import yaml
        cfg = yaml.safe_load(open(args.hyper_path))[args.model]
    for k, v in cfg.items():                                                               # merge_args_config
        if getattr(args, k, None) is None:
            setattr(args, k, v)
    args.output_dim1, args.output_dim2, args.metric_name = 6, 1, "emoval"
    say("args: ", args)
    save_resroot = os.path.join(args.save_root, "result")
    if rank == 0:
        os.makedirs(save_resroot, exist_ok=True)
        os.makedirs(os.path.join(args.save_root, "model"), exist_ok=True)
    feature_name = "+".join(sorted(set(feats)))
    prefix_name = f"features:{feature_name}_dataset:{args.dataset}_model:{args.model}+{args.feat_type}+{args.e2e_name}"

    say("====== Reading Data =======")
    label_path = config.PATH_TO_LABEL[args.dataset]
    names, labels = read_names_labels(label_path, "train", args.debug)
    say(f"train: sample number {len(names)}")
    train_split = DeviceSplit(args, names, labels, config, device)
    folds = random_split_indexes(len(names), 5)
    tests = []
    for dt in ("test1", "test2", "test3"):
        n, l = read_names_labels(label_path, dt, args.debug)
        say(f"{dt}: sample number {len(n)}")
        tests.append(DeviceSplit(args, n, l, config, device))
    train_loaders, eval_loaders, test_loaders = get_loaders(len(names), folds, [len(ts) for ts in tests],
                                                            args.batch_size, args.num_workers)
    args.audio_dim, args.text_dim, args.video_dim = train_split.dims

    say("====== Training and Evaluation =======")
    folder_save, folder_duration = [], []
    name_time = time.time()
    for ii in range(len(train_loaders)):
        say(f">>>>> Cross-validation: training on the {ii + 1} folder >>>>>")
        start_time = name_time = time.time()
        args.seed = random.randint(0, 2 ** 31 - 1)        # dropout-mask stream of this fold's model
        model = get_models(args).cuda()                   # default init from torch's generator, as the reference
        net = model.net
        if world > 1:
            net.broadcast_from(0)
        optimizer = Adam(lr=args.lr, weight_decay=args.l2)
        whole_store, whole_metrics = [], []
        for epoch in range(args.epochs):
            epoch_store = {}
            train_res = run_split(args, net, train_split, train_loaders[ii], optimizer, True, rank, world)
            eval_res = run_split(args, net, train_split, eval_loaders[ii])
            for k, v in eval_res.items():
                epoch_store[f"eval_{k}"] = v
            tm, em = (gain_metric_from_results(r, args.metric_name) for r in (train_res, eval_res))
            whole_metrics.append(em)
            say("epoch:%d; metric:%s; train results:%.4f; eval results:%.4f" % (epoch + 1, args.metric_name, tm, em))
            for jj, ts in enumerate(tests):
                res = run_split(args, net, ts, test_loaders[jj])
                for k, v in res.items():
                    epoch_store[f"test{jj + 1}_{k}"] = v
            whole_store.append(epoch_store)
            if log is not None:
                log.setdefault("train_loss", []).append(float(train_res["loss"]))
                log.setdefault("eval_loss", []).append(float(eval_res["loss"]))
                log.setdefault("test_loss", []).append([float(epoch_store[f"test{j}_loss"]) for j in (1, 2, 3)])
                log.setdefault("train_names", []).append(train_res["names"])
                log.setdefault("eval_names", []).append(eval_res["names"])
        best_index = int(np.argmax(np.array(whole_metrics)))
        folder_save.append(whole_store[best_index])
        folder_duration.append(time.time() - start_time)
        say(f">>>>> Finish: training on the {ii + 1}-th folder, best_index: {best_index}, "
            f"duration: {folder_duration[-1]} >>>>>")
        if log is not None:
            log.setdefault("best_index", []).append(best_index)
        del model, net

    say("====== Prediction and Saving =======")
    if log is not None:
        log["folder_save"] = folder_save
    args.duration = float(np.sum(folder_duration))
    f1 = np.mean([e["eval_emofscore"] for e in folder_save])
    acc = np.mean([e["eval_emoacc"] for e in folder_save])
    mse = np.mean([e["eval_valmse"] for e in folder_save])
    cv_result = f"f1:{f1:.4f}_acc:{acc:.4f}_val:{mse:.4f}"
    saved = []
    path = f"{save_resroot}/cv_{prefix_name}_{cv_result}_{name_time}.npz"
    saved.append(path)
    for jj in range(len(tests)):
        emo_labels = folder_save[0][f"test{jj + 1}_emolabels"]
        emo_probs = np.mean(np.array([f[f"test{jj + 1}_emoprobs"] for f in folder_save]), axis=0)
        val_labels = folder_save[0][f"test{jj + 1}_vallabels"]
        val_preds = np.mean(np.array([f[f"test{jj + 1}_valpreds"] for f in folder_save]), axis=0)
        _, test_result = calculate_results(emo_probs, emo_labels, val_preds, val_labels)
        saved.append(f"{save_resroot}/test{jj + 1}_{prefix_name}_{test_result}_{name_time}.npz")
    if rank == 0:
        for p in saved:
            np.savez_compressed(p, args=np.array(args, dtype=object))
            print(f"save results in {p}")
    return saved


if __name__ == "__main__":
    main(build_parser().parse_args())
