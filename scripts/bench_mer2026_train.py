"""Wall time of a MER2026 Track 1 training run: 5 folds x 100 epochs of ``--model attention`` and of ``--model
attention_topn`` (N = 3, 6, 18 features), emotion-only head, batch 32, hidden 128, dropout 0.3, lr 1e-3, l2 1e-5, on a
synthetic corpus the size of MER2026 Track 1 (9,395 training clips, track1_train.csv; the test1 size is a choice here).

Each epoch is what main_release runs: one training pass over the fold's train part (4/5 of the clips, shuffled by
torch's SubsetRandomSampler), an eval pass over its eval part and a test1 pass.  Two arms on the same GPU, same data,
same loaders:
  ours   FusionNet / TopnFusionNet: one fused training step per batch (CUDA-graph replay for attention, the top-N step
         plus Adam otherwise), eval forwards on the device;
  eager  the repository's torch restatement of the nets (oracle/fusion.py) on the GPU, fp32, with torch.optim.Adam --
         the reference's own loop run in torch eager (the reference tree itself is not available where this runs).
Prints one JSON line per (arm, model) and the card name and power limit beside the numbers; with --out also writes them.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N_TRAIN, N_TEST = 9395, 2000
# the widths of MER2026's ranked extractors, strongest last per list (main_release.RANK_LISTS["MER2026"]):
# HUBERT-base / -large, MacBERT-large / -base, CLIP-large / -base, ...
WIDTHS = [768, 1024, 1024, 768, 768, 512, 1024, 1024, 768, 768, 768, 1024, 256, 512, 512, 1024, 768, 1024]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def make_data(n, widths, seed, dev):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(n, w, generator=g).to(dev) for w in widths]
    emo = torch.randint(0, 6, (n,), generator=g).to(dev)
    return xs, emo


def run(arm, model, n_feats, folds, epochs, dev):
    from mertools_b200 import main_release as MR
    from mertools_b200.fusion import FusionNet, TopnFusionNet, reference_init, reference_init_topn
    from oracle import fusion as OF
    widths = WIDTHS[:3] if model == "attention" else WIDTHS[:n_feats]
    X, emo = make_data(N_TRAIN, widths, 1, dev)
    XT, temo = make_data(N_TEST, widths, 2, dev)
    val = torch.full((N_TRAIN, 0), -10.0, device=dev)
    torch.manual_seed(0)
    import random
    random.seed(0)
    split = MR.random_split_indexes(N_TRAIN, 5)[:folds]
    trl, evl, tel = MR.get_loaders(N_TRAIN, split, [N_TEST], 32)
    H, p = 128, 0.3
    steps = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(folds):
        if model == "attention":
            sd = reference_init("utt", *widths, H, 6, 0)
        else:
            sd = reference_init_topn(widths, H, 6, 0)
        if arm == "ours":
            if model == "attention":
                net = FusionNet(*widths, H, 6, 0, dropout=p, device=dev, max_batch=32, seed=f).load_state_dict(sd)
            else:
                net = TopnFusionNet(widths, H, 6, 0, dropout=p, device=dev, seed=f).load_state_dict(sd)
        else:
            params = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
            opt = torch.optim.Adam(list(params.values()), lr=1e-3, weight_decay=1e-5)

            def fwd(xs, train):
                if not train:
                    masks = None
                else:
                    masks = [(torch.rand_like(x) >= p).float() for x in xs]
                    masks.append((torch.rand(xs[0].shape[0], H * len(xs), device=dev) >= p).float())
                if model == "attention":
                    return OF.attention_forward(params, *xs, masks=masks, p=p)[1]
                return OF.attention_topn_forward(params, xs, masks, p)[1]
        for _ in range(epochs):
            for b in trl[f]:
                b = b.to(dev)
                xs, y = [x.index_select(0, b) for x in X], emo.index_select(0, b)
                if arm == "ours":
                    if model == "attention":
                        net.train_step(*xs, y, val.index_select(0, b), lr=1e-3, weight_decay=1e-5)
                    else:
                        net.train_step(xs, y, val.index_select(0, b), lr=1e-3, weight_decay=1e-5)
                else:
                    opt.zero_grad()
                    loss = torch.nn.functional.cross_entropy(fwd(xs, True), y, reduction="sum") / len(b)
                    loss.backward()
                    opt.step()
                steps += 1
            for loader, XX, yy in ((evl[f], X, emo), (tel[0], XT, temo)):
                probs = []
                for b in loader:
                    b = b.to(dev)
                    xs = [x.index_select(0, b) for x in XX]
                    if arm == "ours":
                        net.train(False)
                        batch = dict(zip(("audios", "texts", "videos"), xs)) if model == "attention" else \
                            {f"feat{i}": x for i, x in enumerate(xs)}
                        eo = net(batch)[1]
                        net.train(True)
                    else:
                        with torch.no_grad():
                            eo = fwd(xs, False)
                    probs.append(eo)
                torch.cat(probs).cpu()  # the host reads the scores every epoch, as the metrics need them
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dict(arm=arm, model=model, n_feats=len(widths), folds=folds, epochs=epochs, train_steps=steps,
                seconds=round(dt, 2), ms_per_train_step_incl_eval=round(dt * 1e3 / steps, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--arms", default="ours,eager")
    ap.add_argument("--models", default="attention,topn3,topn6,topn18")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU: there is no CPU fallback"
    dev = torch.device("cuda:0")
    name, power = card()
    rows = []
    for m in a.models.split(","):
        model, n = ("attention", 3) if m == "attention" else ("attention_topn", int(m[4:]))
        for arm in a.arms.split(","):
            r = run(arm, model, n, a.folds, a.epochs, dev)
            r.update(gpu=name, power_limit=power)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
