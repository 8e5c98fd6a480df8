"""Attention-fusion training CLI — H100 mirror of MERBench/main-release.py for
``--model attention --feat_type utt --dataset MER2023`` (the configuration of SURVEY.md §8 rows
a9-a12), and of the Track 1 trainers of the three later challenges (MER2024/main-release.py,
MER2025/MER2025_Track1/main-release.py, MER2026/MER2026_Track1/main-release.py: one script up to an unused import) for
``--dataset MER2024 | MER2025 | MER2026`` with ``--model attention`` or ``--model attention_topn --fusion_topn n
--fusion_modality AVT | AV | AT | VT``.  Those corpora train an emotion-only head (output_dim2 = 0, metric 'emo',
toolkit/dataloader/mer2026.py:26-28) and have one test set, test1.  Same flags (:93-124), same hyper-parameter handling (model-tune.yaml ``attention`` grid or
``--hyper_path``, :159-165), same label / feature file formats (toolkit/dataloader/mer2023.py:82-104,
toolkit/utils/read_data.py:15-41,92-97), same 5-fold protocol (mer2023.py:108-134), metrics
(toolkit/utils/metric.py) and result files ``cv_*.npz`` / ``test{j}_*.npz`` (:256-272).

What changes is where the work happens: all features live on the GPU once, torch's own ``DataLoader`` /
``SubsetRandomSampler`` only shuffle and batch sample INDICES (so the order of samples and the consumption of
torch's generator are the reference's by construction), batches are index-selected on the device, and every
training step is one fused FusionNet.train_step (forward + CE/MSE + backward + Adam in two kernels).  The golden of
the unmodified script (tests/golden/make_golden_main_release.py) is reproduced fold for fold, epoch for epoch.

The other MERBench corpora follow their own dataloaders (toolkit/dataloader/*.py of MERBench):
``--dataset CMUMOSI | CMUMOSEI | SIMS | SIMSv2`` train a regression-only head (output_dim1 = 0) on train / val / test
and report acc-2 / weighted F1 of the valence sign; ``--dataset MELD`` a 7-class emotion head on train / val / test;
``--dataset IEMOCAPFour | IEMOCAPSix`` a 4- / 6-class head with leave-one-session-out folds and no test set.  The
cross-corpus runs ``--train_dataset X --test_dataset Y`` are crossdim.py (sentiment corpora) and crossdis.py (the four
shared emotions of IEMOCAP, MER2023 and MELD).

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
from .fusion import Adam, get_models, mer2023_calculate_results, mer2026_calculate_results, sentiment_calculate_results

EMOS_MER = ["neutral", "angry", "happy", "sad", "worried", "surprise"]      # toolkit/globals.py:2
EMO2IDX = {e: i for i, e in enumerate(EMOS_MER)}
ATTENTION_GRID = dict(hidden_dim=[64, 128, 256], dropout=[0.2, 0.3, 0.4, 0.5], grad_clip=[-1.0],
                      lr=[1e-3, 1e-4])                                       # toolkit/model-tune.yaml:76-80
# the attention_topn entry of model-tune.yaml:108-112 in the MER2024, MER2025_Track1 and MER2026_Track1 trees
TOPN_GRID = dict(hidden_dim=[64, 128, 256], dropout=[0.2, 0.3, 0.4, 0.5], grad_clip=[-1.0], lr=[1e-3, 1e-4])

# Corpora whose dataloaders (toolkit/dataloader/mer2024.py, mer2025.py, mer2026.py; identical up to the name) read
# train_corpus / test1_corpus, label every clip {'emo': idx, 'val': -10} and set output_dim1 = 6, output_dim2 = 0,
# metric_name = 'emo'.
EMO_CORPORA = ("MER2024", "MER2025", "MER2026")
# The sentiment corpora (DIM_DATASET, toolkit/dataloader/__init__.py:10): cmudata.py:20-23, sims.py:21-23, simsv2.py:21-24
# and crossdim.py:19-21 set output_dim1 = 0, output_dim2 = 1, metric_name = 'emo' and read train / val / test.
SENTIMENT_CORPORA = ("CMUMOSI", "CMUMOSEI", "SIMS", "SIMSv2")
# The corpora crossdis.py trains and tests across (DIS_DATASET, toolkit/dataloader/__init__.py:11).
CROSSDIS_CORPORA = ("IEMOCAPFour", "IEMOCAPSix", "MER2023", "MELD")
IEMOCAP_CORPORA = ("IEMOCAPFour", "IEMOCAPSix")
# (output_dim1, output_dim2, metric_name) per --dataset: mer2023.py, mer2026.py:26-28, iemocap.py:25-33, meld.py:20-22
# and the sentiment loaders above.
HEADS = {"MER2023": (6, 1, "emoval"), **{d: (6, 0, "emo") for d in EMO_CORPORA},
         **{d: (0, 1, "emo") for d in SENTIMENT_CORPORA}, "IEMOCAPFour": (4, 0, "emo"), "IEMOCAPSix": (6, 0, "emo"),
         "MELD": (7, 0, "emo")}
# crossdis.py:9-16: the four shared emotions and each corpus' label -> emotion map (samples outside it are dropped)
CROSSDIS_EMO2IDX = {"happy": 0, "sad": 1, "neutral": 2, "angry": 3}
CROSSDIS_MAP = {
    "IEMOCAPFour": {0: "happy", 1: "sad", 2: "neutral", 3: "angry"},
    "IEMOCAPSix": {0: "happy", 1: "sad", 2: "neutral", 3: "angry"},
    "MELD": {0: "angry", 1: "happy", 2: "sad", 3: "neutral"},
    "MER2023": {"neutral": "neutral", "angry": "angry", "happy": "happy", "sad": "sad"},
}

# Feature rankings, weakest first, that Data_Feat_TOPN takes the top n of (toolkit/globals.py of each tree):
#   MER2024/toolkit/globals.py:218-231, MER2025/MER2025_Track1/toolkit/globals.py:218-242,
#   MER2026/MER2026_Track1/toolkit/globals.py:218-240.
RANK_LISTS = {
    "MER2024": dict(
        audio=["eGeMAPS", "VGGish", "Whisper-base", "emotion2vec", "Whisper-large", "wav2vec 2.0-base",
               "wav2vec 2.0-large", "HUBERT-base", "HUBERT-large"],
        text=["XLNet-base", "ELECTRA-large", "MOSS-7B", "PERT-large", "PERT-base", "LERT-large", "ELECTRA-base",
              "LERT-base", "RoBERTa-base", "MacBERT-base", "RoBERTa-large", "ChatGLM2-6B", "MacBERT-large", "BLOOM-7B",
              "Baichuan-13B"],
        image=["VideoMAE-base", "EmoNet", "VideoMAE-large", "DINOv2-large", "SENet-FER2013", "ResNet-FER2013",
               "MANet-RAFDB", "EVA-02-base", "CLIP-base", "VideoMAE-base (VoxCeleb2)", "VideoMAE-base (MER2023)",
               "CLIP-large"]),
    "MER2025": dict(
        audio=["WavLM-base", "wav2vec 2.0-large", "wav2vec 2.0-base", "Whisper-large", "HUBERT-base", "HUBERT-large"],
        text=["MacBERT-base", "MacBERT-large", "BLOOM-7B", "RoBERTa-large", "RoBERTa-base"],
        image=["ResNet-FER2013", "DINOv2-large", "SENet-FER2013", "MANet-RAFDB", "CLIP-base", "CLIP-large"]),
    "MER2026": dict(
        audio=["WavLM-base", "wav2vec 2.0-base", "wav2vec 2.0-large", "HUBERT-large", "HUBERT-base"],
        text=["RoBERTa-base", "RoBERTa-large", "MacBERT-base", "MacBERT-large"],
        image=["VideoMAE-large", "ResNet-FER2013", "EmoNet", "SENet-FER2013", "CLIP-base", "CLIP-large"]),
}
# The display name -> feature directory entries of featname_mapping (toolkit/globals.py:145-203, the same in the
# three trees) that the rank lists above use.
FEATNAME_DIRS = {
    "BLOOM-7B": "bloom-7b1", "Baichuan-13B": "Baichuan-13B-Base", "CLIP-base": "clip-vit-base-patch32",
    "CLIP-large": "clip-vit-large-patch14", "ChatGLM2-6B": "chatglm2-6b", "DINOv2-large": "dinov2-large",
    "ELECTRA-base": "chinese-electra-180g-base", "ELECTRA-large": "chinese-electra-180g-large",
    "EVA-02-base": "eva02_base_patch14_224", "EmoNet": "emonet", "HUBERT-base": "chinese-hubert-base",
    "HUBERT-large": "chinese-hubert-large", "LERT-base": "chinese-lert-base", "LERT-large": "chinese-lert-large",
    "MANet-RAFDB": "manet", "MOSS-7B": "moss-base-7b", "MacBERT-base": "chinese-macbert-base",
    "MacBERT-large": "chinese-macbert-large", "PERT-base": "chinese-pert-base", "PERT-large": "chinese-pert-large",
    "ResNet-FER2013": "resnet50face", "RoBERTa-base": "chinese-roberta-wwm-ext",
    "RoBERTa-large": "chinese-roberta-wwm-ext-large", "SENet-FER2013": "senet50face", "VGGish": "vggish",
    "VideoMAE-base": "videomae-base", "VideoMAE-base (MER2023)": "videomae-base-K400-mer2023-299",
    "VideoMAE-base (VoxCeleb2)": "videomae-base-VoxCeleb2-99", "VideoMAE-large": "videomae-large",
    "WavLM-base": "wavlm-base", "Whisper-base": "whisper-base", "Whisper-large": "whisper-large-v2",
    "XLNet-base": "chinese-xlnet-base", "eGeMAPS": "eGeMAPS", "emotion2vec": "emotion2vec",
    "wav2vec 2.0-base": "chinese-wav2vec2-base", "wav2vec 2.0-large": "chinese-wav2vec2-large",
}
# Data_Feat_TOPN's RANK_LIST per --fusion_modality (toolkit/data/feat_data_topn.py:16-24): three lists, not one per
# modality -- AT takes the text ranking twice, AV the image ranking twice, VT text twice then image.
FUSION_MODALITIES = {"AVT": ("audio", "text", "image"), "AT": ("audio", "text", "text"),
                     "AV": ("audio", "image", "image"), "VT": ("text", "text", "image")}


def func_name_conversion(display_name, feature_root, suffix="UTT"):
    """toolkit/utils/functions.py:329-336 (MER2025 / MER2026): ``<dir>_UTT`` when that directory exists under the
    corpus' feature root, otherwise ``<dir>-UTT``.  MER2024's copy (functions.py:246-253) looks under
    config.PATH_TO_FEATURES['SIMS'] whatever the corpus; here every corpus looks under its own feature root, which is
    what the MER2025 / MER2026 copies do and the only root that holds MER2024's features."""
    d = FEATNAME_DIRS[display_name]
    return f"{d}_{suffix}" if os.path.exists(os.path.join(feature_root, f"{d}_{suffix}")) else f"{d}-{suffix}"


def topn_feature_names(dataset, fusion_topn, fusion_modality, feature_root):
    """Data_Feat_TOPN (toolkit/data/feat_data_topn.py:16-31): the last ``fusion_topn`` names of each of the three
    rank lists, in list order, resolved to feature directories -> 3 * fusion_topn names (repeats included)."""
    assert fusion_topn is not None and fusion_modality in FUSION_MODALITIES, (fusion_topn, fusion_modality)
    assert 1 <= fusion_topn, fusion_topn
    names = []
    for which in FUSION_MODALITIES[fusion_modality]:
        names.extend(RANK_LISTS[dataset][which][-fusion_topn:])
    assert len(names) == 3 * fusion_topn, f"a rank list of {dataset} is shorter than --fusion_topn {fusion_topn}"
    return [func_name_conversion(n, feature_root) for n in names]


# ---- data (host side, same file formats as the reference) ---------------------------------------
SPLITS = {"MER2023": ("train", "test1", "test2", "test3"), **{d: ("train", "test1") for d in EMO_CORPORA},
          **{d: ("train", "val", "test") for d in SENTIMENT_CORPORA + ("MELD",)},
          **{d: ("whole",) for d in IEMOCAP_CORPORA}}


def read_names_labels(label_path, data_type, debug=False, dataset="MER2023"):
    """mer2023.py:82-104; for MER2024 / 25 / 26 mer2026.py:83-99 (train / test1 only, the valence is always -10); for
    the sentiment corpora and MELD cmudata.py:58-70 / sims.py / simsv2.py / meld.py:56-68 (train / val / test), for
    IEMOCAP iemocap.py:64-75 (whole): those labels are stored as the loaders use them (an integer emotion, a float
    valence) and are passed through."""
    assert data_type in SPLITS[dataset], (dataset, data_type)
    corpus = np.load(label_path, allow_pickle=True)[f"{data_type}_corpus"].tolist()
    names, labels = [], []
    for name, label in corpus.items():
        names.append(name)
        if dataset in EMO_CORPORA:
            labels.append({"emo": EMO2IDX[label["emo"]], "val": -10})
        elif dataset == "MER2023":
            val = label["val"] if ("val" in label and label["val"] != "") else -10
            labels.append({"emo": EMO2IDX[label["emo"]], "val": val})
        else:
            labels.append({"emo": int(label["emo"]), "val": label["val"]})
    if debug:
        names, labels = names[:100], labels[:100]
    return names, labels


def read_crossdim_labels(label_path, dataset, data_type, debug=False):
    """crossdim.py:66-83: a sentiment corpus' split with the SIMS / SIMSv2 valences (in [-1, 1]) scaled by 3 to the CMU
    range [-3, 3]."""
    assert dataset in SENTIMENT_CORPORA, dataset
    names, labels = read_names_labels(label_path, data_type, False, dataset)
    if dataset in ("SIMS", "SIMSv2"):
        for l in labels:
            l["val"] = l["val"] * 3
    if debug:
        names, labels = names[:100], labels[:100]
    return names, labels


def read_crossdis_labels(label_path, dataset, data_type, debug=False):
    """crossdis.py:162-188: a split mapped onto the four shared emotions (CROSSDIS_MAP then CROSSDIS_EMO2IDX), the
    samples whose emotion is outside the map dropped; the valence is passed through (-10 where the corpus has none)."""
    assert dataset in CROSSDIS_CORPORA, dataset
    assert data_type in {"MER2023": ("train", "test1"), "MELD": ("train", "val", "test")}.get(dataset, ("whole",)), \
        (dataset, data_type)
    corpus = np.load(label_path, allow_pickle=True)[f"{data_type}_corpus"].tolist()
    mapping = CROSSDIS_MAP[dataset]
    names, labels = [], []
    for name, label in corpus.items():
        if label["emo"] in mapping:
            names.append(name)
            val = label.get("val", -10)
            labels.append({"emo": CROSSDIS_EMO2IDX[mapping[label["emo"]]], "val": -10 if val == "" else val})
    if debug:
        names, labels = names[:100], labels[:100]
    return names, labels


def session_split_indexes(names, num_folder=5):
    """iemocap.py:78-96 / crossdis.py:191-203: leave-one-session-out -- fold i evaluates session i + 1
    (``int(name[4]) - 1``: ``Ses0N...``) and trains on the other four, each in corpus order."""
    session_to_idx = {}
    for idx, vid in enumerate(names):
        session_to_idx.setdefault(int(vid[4]) - 1, []).append(idx)
    assert len(session_to_idx) == num_folder, "Must split into five folder"
    return [[[i for j in range(num_folder) if j != k for i in session_to_idx[j]], list(session_to_idx[k])]
            for k in range(num_folder)]


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
    frame-level types (shaped exactly as Data_Feat does, feat_data.py:33-44) -- emo int64, val fp32.  For
    attention_topn: the 3 * fusion_topn utterance-level features ``args.topn_features`` (Data_Feat_TOPN: the mean over
    time of each clip), as ``feats``."""

    def __init__(self, args, names, labels, config, device, dataset=None):
        root = config.PATH_TO_FEATURES[dataset or args.dataset]     # each corpus' own features (feat_data.py:12)
        feats = []
        if args.model == "attention_topn":
            for fname in args.topn_features:
                fr = os.path.join(root, fname)
                feats.append(np.stack([read_utt_feature(fr, n) for n in names]).astype(np.float32))
        elif args.feat_type == "utt":
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
        self.feats = [torch.from_numpy(f).to(device) for f in feats]
        if args.model != "attention_topn":
            self.a, self.t, self.v = self.feats
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


def sequential_loader(n, batch_size, num_workers=0):
    """The train, val and test loaders of cmudata.py:29-52 (and sims.py, simsv2.py, meld.py, crossdim.py, crossdis.py's
    MELD branch): no shuffle, no sampler -- the split in corpus order.  Iterating it still draws the loader's base seed
    from torch's generator, as the reference's does."""
    from torch.utils.data import DataLoader
    return DataLoader(_Indices(n), batch_size=batch_size, num_workers=num_workers, shuffle=False)


calculate_results = mer2023_calculate_results  # mer2023.py:137-155


def corpus_calculate_results(dataset, train_dataset=None):
    """dataloader_class.calculate_results: mer2023.py:137-155; the argmax f1 / acc rule of mer2026.py:132-145 for
    MER2024 / 25 / 26, which is also iemocap.py:99-115, meld.py:72-87 and crossdis.py:228-243; acc-2 of the valence
    sign (cmudata.py:69-84, crossdim.py:87-102) for the sentiment corpora.  A cross-corpus run takes the rule of its
    protocol, chosen by the train corpus (toolkit/dataloader/__init__.py:32-37)."""
    if train_dataset is not None:
        return sentiment_calculate_results if train_dataset in SENTIMENT_CORPORA else mer2026_calculate_results
    if dataset in SENTIMENT_CORPORA:
        return sentiment_calculate_results
    return mer2023_calculate_results if dataset == "MER2023" else mer2026_calculate_results


def gain_cv_results(folder_save):
    """toolkit/utils/metric.py:35-54: the means over the folds' best epochs of the eval metrics that are present."""
    keys = folder_save[0].keys()
    out = []
    for key, label in (("eval_emofscore", "f1"), ("eval_emoacc", "acc"), ("eval_valmse", "val")):
        if key in keys:
            out.append(f"{label}:{np.mean([e[key] for e in folder_save]):.4f}")
    return "_".join(out)


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


def load_protocol(args, config, device, say=print):
    """The splits and loader objects of the corpus' dataloader class (toolkit/dataloader/__init__.py:14-37), in the order
    the reference builds them.  Returns (folds, tests, train_loaders, eval_loaders, test_loaders): ``folds[i]`` is the
    (train, eval) pair of DeviceSplits fold i's loaders index into, ``tests`` the test DeviceSplits."""
    bs, nw = args.batch_size, args.num_workers
    mk = lambda names, labels, ds: DeviceSplit(args, names, labels, config, device, ds)  # noqa: E731
    seq = lambda split: sequential_loader(len(split), bs, nw)  # noqa: E731
    if args.train_dataset is not None:
        return _load_cross(args, config, mk, seq, say)
    ds = args.dataset
    lp = config.PATH_TO_LABEL[ds]
    if ds in IEMOCAP_CORPORA:                     # iemocap.py:35-61: five session folds over whole_corpus, no test set
        names, labels = read_names_labels(lp, "whole", args.debug, ds)
        folds = session_split_indexes(names)
        say(f"sample number {len(names)}")
        whole = mk(names, labels, ds)
        trl, evl, _ = get_loaders(len(names), folds, [], bs, nw)
        return [(whole, whole)] * len(folds), [], trl, evl, []
    if ds in SENTIMENT_CORPORA or ds == "MELD":   # cmudata.py:26-55 / sims.py / simsv2.py / meld.py: one fold
        splits = []
        for dt in ("train", "val", "test"):
            names, labels = read_names_labels(lp, dt, args.debug, ds)
            say(f"{dt}: sample number {len(names)}")
            splits.append(mk(names, labels, ds))
        return [(splits[0], splits[1])], [splits[2]], [seq(splits[0])], [seq(splits[1])], [seq(splits[2])]
    # MER2023 (mer2023.py:31-79), MER2024 / 25 / 26 (mer2026.py:31-80): five random folds of train, then the test sets
    names, labels = read_names_labels(lp, "train", args.debug, ds)
    say(f"train: sample number {len(names)}")
    train_split = mk(names, labels, ds)
    folds = random_split_indexes(len(names), 5)
    tests = []
    for dt in SPLITS[ds][1:]:
        n, l = read_names_labels(lp, dt, args.debug, ds)
        say(f"{dt}: sample number {len(n)}")
        tests.append(mk(n, l, ds))
    trl, evl, tel = get_loaders(len(names), folds, [len(ts) for ts in tests], bs, nw)
    return [(train_split, train_split)] * len(folds), tests, trl, evl, tel


def _load_cross(args, config, mk, seq, say):
    """crossdim.py:23-56 (sentiment corpora: train / val of the train corpus, test of the test corpus, one fold) and
    crossdis.py:33-139 (IEMOCAP: session folds of whole; MER2023: five random folds of train; MELD: train / val; then
    the test split of the test corpus: whole, test1 or test).  Each split reads its own corpus' features."""
    tr, te = args.train_dataset, args.test_dataset
    assert te is not None, "--train_dataset needs --test_dataset"
    if tr in SENTIMENT_CORPORA:
        assert te in SENTIMENT_CORPORA, f"crossdim tests on {SENTIMENT_CORPORA}, not {te}"
        s = []
        for ds, dt in ((tr, "train"), (tr, "val"), (te, "test")):
            names, labels = read_crossdim_labels(config.PATH_TO_LABEL[ds], ds, dt, args.debug)
            say(f"{dt}: sample number {len(names)}")
            s.append(mk(names, labels, ds))
        return [(s[0], s[1])], [s[2]], [seq(s[0])], [seq(s[1])], [seq(s[2])]
    assert tr in CROSSDIS_CORPORA and te in CROSSDIS_CORPORA, \
        f"cross-corpus runs pair {SENTIMENT_CORPORA} or {CROSSDIS_CORPORA}, not {tr} -> {te}"
    rd = lambda ds, dt: read_crossdis_labels(config.PATH_TO_LABEL[ds], ds, dt, args.debug)  # noqa: E731
    if tr in IEMOCAP_CORPORA:
        names, labels = rd(tr, "whole")
        folds = session_split_indexes(names)
        whole = mk(names, labels, tr)
        pairs = [(whole, whole)] * len(folds)
        trl, evl, _ = get_loaders(len(names), folds, [], args.batch_size, args.num_workers)
    elif tr == "MER2023":
        names, labels = rd(tr, "train")
        whole = mk(names, labels, tr)
        folds = random_split_indexes(len(names), 5)
        pairs = [(whole, whole)] * len(folds)
        trl, evl, _ = get_loaders(len(names), folds, [], args.batch_size, args.num_workers)
    else:
        train, val = mk(*rd(tr, "train"), tr), mk(*rd(tr, "val"), tr)
        pairs, trl, evl = [(train, val)], [seq(train)], [seq(val)]
    test = mk(*rd(te, {"MER2023": "test1", "MELD": "test"}.get(te, "whole")), te)
    say(f"test: sample number {len(test)}")
    return pairs, [test], trl, evl, [seq(test)]


# ---- one pass over a split (main-release.py:17-87) ------------------------------------------------
def run_split(args, net, split, loader, optimizer=None, train=False, rank=0, world_size=1):
    """``loader`` yields batches of sample indices in the reference's order.  Training: one fused step per batch
    (under data parallelism on rows ``rank::world_size`` of it); evaluation: eval forward + the losses.  The CE loss
    and the emotion scores enter only when ``args.output_dim1 != 0``, the regression loss and the valence predictions
    only when ``args.output_dim2 != 0`` (main-release.py:51-58)."""
    dev = split.emo.device
    topn = args.model == "attention_topn"
    has_emo, has_val = args.output_dim1 != 0, args.output_dim2 != 0
    names, emo_probs, val_preds, losses, order = [], [], [], [], []
    net.train(train)
    for b in loader:
        names += [split.names[i] for i in b.tolist()]
        b = b.to(dev)
        order.append(b)
        mine = b[rank::world_size] if (train and world_size > 1) else b
        xs = [f.index_select(0, mine) for f in split.feats]
        emo, val = split.emo.index_select(0, mine), split.val.index_select(0, mine)
        if train:
            kw = dict(lr=optimizer.lr, betas=optimizer.betas, eps=optimizer.eps, weight_decay=optimizer.weight_decay,
                      world_size=world_size, global_batch=len(b))
            loss3, eo, vo = net.train_step(xs, emo, val, **kw) if topn else net.train_step(*xs, emo, val, **kw)
            losses.append(loss3[2:3].clone())
            if world_size > 1:
                if has_emo:
                    eo = _gather_strided(eo, len(b), rank, world_size)
                if has_val:
                    vo = _gather_strided(vo, len(b), rank, world_size)
        else:
            batch = {f"feat{i}": x for i, x in enumerate(xs)} if topn else dict(zip(("audios", "texts", "videos"), xs))
            _, eo, vo, _ = net(batch)
            loss = torch.zeros(1, device=dev)
            if has_emo:
                loss = loss + torch.nn.functional.cross_entropy(eo, emo, reduction="sum") / len(eo)
            if has_val:
                loss = loss + torch.nn.functional.mse_loss(vo, val, reduction="sum") / len(vo)
            losses.append(loss.view(1))
        if has_emo:
            emo_probs.append(eo.clone())
        if has_val:
            val_preds.append(vo.clone())
    order = torch.cat(order)
    emo_labels, val_labels = [], []
    if has_emo:
        emo_probs = torch.cat(emo_probs).cpu().numpy()
        emo_labels = split.emo.index_select(0, order).cpu().numpy()
    if has_val:
        val_preds = torch.cat(val_preds).cpu().numpy()
        val_labels = split.val.index_select(0, order).cpu().numpy()
    res, _ = corpus_calculate_results(args.dataset, getattr(args, "train_dataset", None))(
        emo_probs, emo_labels, val_preds, val_labels)
    return dict(names=names, loss=np.mean(torch.cat(losses).cpu().numpy()), **res)


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--dataset", type=str, default=None)          # MER2023 unless a cross-corpus run
    p.add_argument("--train_dataset", type=str, default=None)    # cross-corpus runs (main-release.py:96-97)
    p.add_argument("--test_dataset", type=str, default=None)
    p.add_argument("--fusion_topn", type=int, default=None)
    p.add_argument("--fusion_modality", type=str, default="AVT")
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


def result_prefix(args):
    """prefix_name of the result files (main-release.py:170-179).  The reference builds it before its loaders run, so
    the dataset: field is --dataset as given -- None in a cross-corpus run that passes only --train_dataset /
    --test_dataset."""
    feats = [f for f in (args.audio_feature, args.text_feature, args.video_feature) if f is not None]
    prefix = (f"features:{'+'.join(sorted(set(feats)))}_dataset:{args.dataset}_model:{args.model}+{args.feat_type}+"
              f"{args.e2e_name}")
    if args.fusion_topn is not None:
        prefix += f"_fusiontopn:{args.fusion_topn}_modality:{args.fusion_modality}"
    if getattr(args, "train_dataset", None) is not None:
        prefix += f"_train:{args.train_dataset}_test:{args.test_dataset}"
    return prefix


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
    cross = getattr(args, "train_dataset", None) is not None
    if not cross:
        args.train_dataset = args.test_dataset = None
        if args.dataset is None:
            args.dataset = "MER2023"
        assert args.dataset in HEADS, f"the H100 path covers --dataset {' / '.join(HEADS)}, not {args.dataset}"
    assert args.model == "attention" or (args.model == "attention_topn" and args.dataset in EMO_CORPORA and not cross), \
        "the H100 path covers --model attention, and attention_topn on the corpora with feature rankings"
    topn = args.model == "attention_topn"
    rank, world = _init_distributed(args)
    torch.cuda.set_device(args.gpu)
    device = torch.device("cuda", args.gpu)
    say = print if rank == 0 else (lambda *a, **k: None)
    # pre-compression of the frame-level types (main-release.py:131-142)
    if topn:
        assert args.feat_type == "utt", "attention_topn reads utterance-level features (feat_data_topn.py:36-39)"
    if args.feat_type == "utt":
        args.feat_scale = 1
    else:
        assert args.feat_type in ("frm_align", "frm_unalign"), args.feat_type
        for f in (args.audio_feature, args.text_feature, args.video_feature):
            assert f.endswith("FRA"), f"feat_type {args.feat_type} needs frame-level features, got {f}"
        args.feat_scale = 6 if args.feat_type == "frm_align" else 12
    if args.fusion_topn is not None:
        args.save_root = f"{args.save_root}-multitop"
    if cross:
        args.save_root = f"{args.save_root}-cross"
    feats = [f for f in (args.audio_feature, args.text_feature, args.video_feature) if f is not None]
    args.save_root = f"{args.save_root}-" + {0: "others", 1: "unimodal", 2: "bimodal", 3: "trimodal"}[len(set(feats))]
    if args.hyper_path is None:
        grid = TOPN_GRID if topn else ATTENTION_GRID
        cfg = {k: v[random.randint(0, len(v) - 1)] for k, v in grid.items()}              # func_random_select
    else:
        import yaml
        cfg = yaml.safe_load(open(args.hyper_path))[args.model]
    for k, v in cfg.items():                                                               # merge_args_config
        if getattr(args, k, None) is None:
            setattr(args, k, v)
    if cross:   # crossdim.py:19-21 / crossdis.py:29-31
        args.output_dim1, args.output_dim2, args.metric_name = (0, 1, "emo") if args.train_dataset in SENTIMENT_CORPORA \
            else (4, 0, "emo")
    else:
        args.output_dim1, args.output_dim2, args.metric_name = HEADS[args.dataset]
    say("args: ", args)
    save_resroot = os.path.join(args.save_root, "result")
    if rank == 0:
        os.makedirs(save_resroot, exist_ok=True)
        os.makedirs(os.path.join(args.save_root, "model"), exist_ok=True)
    prefix_name = result_prefix(args)

    say("====== Reading Data =======")
    if topn:
        args.topn_features = topn_feature_names(args.dataset, args.fusion_topn, args.fusion_modality,
                                                config.PATH_TO_FEATURES[args.dataset])
        say(f"feature number: {len(args.topn_features)}")
    folds, tests, train_loaders, eval_loaders, test_loaders = load_protocol(args, config, device, say)
    if cross:   # the cross-corpus loaders leave args.dataset at the test corpus (crossdim.py:36, crossdis.py:122)
        args.dataset = args.test_dataset
    say(f"train&val folder:{len(train_loaders)}; test sets:{len(test_loaders)}")
    if topn:  # Data_Feat_TOPN.get_featdim: the list of widths, three times
        args.audio_dim = args.text_dim = args.video_dim = list(folds[0][0].dims)
    else:
        args.audio_dim, args.text_dim, args.video_dim = folds[0][0].dims

    say("====== Training and Evaluation =======")
    folder_save, folder_duration = [], []
    name_time = time.time()
    for ii in range(len(train_loaders)):
        say(f">>>>> Cross-validation: training on the {ii + 1} folder >>>>>")
        start_time = name_time = time.time()
        args.seed = random.randint(0, 2 ** 31 - 1)        # dropout-mask stream of this fold's model
        model = get_models(args).cuda()                   # default init from torch's generator, as the reference
        net = model.model if topn else model.net
        if world > 1:
            net.broadcast_from(0)
        optimizer = Adam(lr=args.lr, weight_decay=args.l2)
        whole_store, whole_metrics = [], []
        for epoch in range(args.epochs):
            epoch_store = {}
            train_res = run_split(args, net, folds[ii][0], train_loaders[ii], optimizer, True, rank, world)
            eval_res = run_split(args, net, folds[ii][1], eval_loaders[ii])
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
                log.setdefault("test_loss", []).append([float(epoch_store[f"test{j + 1}_loss"])
                                                        for j in range(len(tests))])
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
    cv_result = gain_cv_results(folder_save)
    saved, contents = [], []
    path = f"{save_resroot}/cv_{prefix_name}_{cv_result}_{name_time}.npz"
    saved.append(path)
    contents.append({})
    for jj in range(len(tests)):   # average_folder_for_emos / _vals (metric.py:57-100): [] when the head is absent
        emo_labels, emo_probs, val_labels, val_preds = [], [], [], []
        if args.output_dim1 != 0:
            emo_labels = folder_save[0][f"test{jj + 1}_emolabels"]
            emo_probs = np.mean(np.array([f[f"test{jj + 1}_emoprobs"] for f in folder_save]), axis=0)
        if args.output_dim2 != 0:
            val_labels = folder_save[0][f"test{jj + 1}_vallabels"]
            val_preds = np.mean(np.array([f[f"test{jj + 1}_valpreds"] for f in folder_save]), axis=0)
        _, test_result = corpus_calculate_results(args.dataset, args.train_dataset)(emo_probs, emo_labels, val_preds,
                                                                                    val_labels)
        saved.append(f"{save_resroot}/test{jj + 1}_{prefix_name}_{test_result}_{name_time}.npz")
        # MER2024 / 25 / 26 keep the fold-averaged emotion scores (MER2026_Track1/main-release.py:286-288)
        contents.append(dict(emo_probs=emo_probs) if args.dataset in EMO_CORPORA else {})
    if rank == 0:
        for p, extra in zip(saved, contents):
            np.savez_compressed(p, **extra, args=np.array(args, dtype=object))
            print(f"save results in {p}")
    return saved


if __name__ == "__main__":
    main(build_parser().parse_args())
