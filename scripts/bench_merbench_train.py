"""Wall time of MERBench training runs beyond MER2023, on synthetic corpora of realistic size:
  sentiment  the CMU-MOSEI protocol (cmudata.py): regression-only head (output_dim1 = 0, MSE alone), one fold, the
             train split in corpus order (no shuffle), then a val and a test pass per epoch.  Sizes: CMU-MOSEI's split
             sizes, 16,326 train / 1,871 val / 4,659 test clips.
  iemocap    the IEMOCAPFour protocol (iemocap.py): 4-class head (output_dim2 = 0, CE alone), leave-one-session-out
             folds over the whole corpus with SubsetRandomSampler for train and eval, no test set.  Size: 5,531 clips
             (IEMOCAP's four-class corpus) in five sessions of about 1,100.
Batch 32, hidden 128, dropout 0.3, lr 1e-3, l2 1e-5; A / T / V widths 1024 / 1024 / 768 (HUBERT-large, a large text
encoder, CLIP-large).  Each epoch is what main_release runs for the protocol.  Two arms on the same GPU, same data, same
loaders:
  ours   FusionNet: one fused training step per batch (CUDA-graph replay), eval forwards on the device;
  eager  the repository's torch restatement of the net (oracle/fusion.py) on the GPU, fp32, with torch.optim.Adam --
         the reference's own loop run in torch eager (the reference tree itself is not available where this runs).
Prints one JSON line per (protocol, arm) with the card name and power limit beside the numbers; --out also writes them.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__))))

from bench_mer2026_train import card  # noqa: E402

WIDTHS = (1024, 1024, 768)
SENTIMENT = (16326, 1871, 4659)
IEMOCAP = 5531


def make_data(n, out1, seed, dev):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(n, w, generator=g).to(dev) for w in WIDTHS]
    emo = torch.randint(0, max(out1, 1), (n,), generator=g).to(dev)
    val = (torch.randint(-9, 10, (n, 1), generator=g).float() / 3).to(dev)
    return xs, emo, val


def run(arm, protocol, folds, epochs, dev):
    from mertools_b200 import main_release as MR
    from mertools_b200.fusion import FusionNet, reference_init
    from oracle import fusion as OF
    torch.manual_seed(0)
    if protocol == "sentiment":
        out1, out2 = 0, 1
        splits = [make_data(n, out1, s, dev) for s, n in enumerate(SENTIMENT)]
        trl = [MR.sequential_loader(SENTIMENT[0], 32)]
        evals = [[(MR.sequential_loader(n, 32), s) for n, s in zip(SENTIMENT[1:], splits[1:])]]
        train = [splits[0]]
    else:
        out1, out2 = 4, 0
        whole = make_data(IEMOCAP, out1, 0, dev)
        names = [f"Ses0{1 + (i * 7) % 5}F_{i:05d}" for i in range(IEMOCAP)]
        tr, ev, _ = MR.get_loaders(IEMOCAP, MR.session_split_indexes(names), [], 32)
        trl, evals, train = tr, [[(e, whole)] for e in ev], [whole] * 5
    folds = min(folds, len(trl))
    H, p = 128, 0.3
    steps = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(folds):
        sd = reference_init("utt", *WIDTHS, H, out1, out2)
        X, emo, val = train[f]
        if arm == "ours":
            net = FusionNet(*WIDTHS, H, out1, out2, dropout=p, device=dev, max_batch=32, seed=f).load_state_dict(sd)
        else:
            params = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
            opt = torch.optim.Adam(list(params.values()), lr=1e-3, weight_decay=1e-5)

            def fwd(xs, training):
                masks = None
                if training:
                    masks = [(torch.rand_like(x) >= p).float() for x in xs]
                    masks.append((torch.rand(xs[0].shape[0], 3 * H, device=dev) >= p).float())
                return OF.attention_forward(params, *xs, masks=masks, p=p)
        for _ in range(epochs):
            for b in trl[f]:
                b = b.to(dev)
                xs, y, v = [x.index_select(0, b) for x in X], emo.index_select(0, b), val.index_select(0, b)
                if arm == "ours":
                    net.train_step(*xs, y, v if out2 else v[:, :0], lr=1e-3, weight_decay=1e-5)
                else:
                    opt.zero_grad()
                    _, eo, vo = fwd(xs, True)
                    if out1:
                        loss = torch.nn.functional.cross_entropy(eo, y, reduction="sum") / len(b)
                    else:
                        loss = torch.nn.functional.mse_loss(vo, v, reduction="sum") / len(b)
                    loss.backward()
                    opt.step()
                steps += 1
            for loader, (XX, _, _) in evals[f]:
                outs = []
                for b in loader:
                    b = b.to(dev)
                    xs = [x.index_select(0, b) for x in XX]
                    if arm == "ours":
                        net.train(False)
                        _, eo, vo, _ = net(dict(zip(("audios", "texts", "videos"), xs)))
                        net.train(True)
                    else:
                        with torch.no_grad():
                            _, eo, vo = fwd(xs, False)
                    outs.append(eo if out1 else vo)
                torch.cat(outs).cpu()  # the host reads the predictions every epoch, as the metrics need them
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dict(arm=arm, protocol=protocol, out1=out1, out2=out2, folds=folds, epochs=epochs, train_steps=steps,
                seconds=round(dt, 2), ms_per_train_step_incl_eval=round(dt * 1e3 / steps, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folds", type=int, default=1)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--arms", default="ours,eager")
    ap.add_argument("--protocols", default="sentiment,iemocap")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU: there is no CPU fallback"
    dev = torch.device("cuda:0")
    name, power = card()
    rows = []
    for protocol in a.protocols.split(","):
        for arm in a.arms.split(","):
            run(arm, protocol, 1, 1, dev)   # warm-up: torch's first-use set-up, the CUDA graph capture
            r = run(arm, protocol, a.folds, a.epochs, dev)
            r.update(gpu=name, power_limit=power)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
