"""Throughput of the ALBERT text-feature path at the five published shapes (albert_chinese_tiny / _small,
albert-base / large / xxlarge-v2) against the reference's loop.

Packed path: AlbertNet on the CUDA backend with BertEncoder's operand rule (f16 up to 768, bf16x3 above), sentences
packed up to --tokens per pass.  Reference loop (extract_text_huggingface.py): HF AlbertModel in fp32 at batch 1,
output_hidden_states and the last-four sum.  Weights are seeded random fp32 tensors (synthetic.albert_state_dict);
sentence lengths are bench_llm_text.py's seeded draws, capped at 512 tokens.  Time shares of GEMM / attention /
LayerNorm / split come from CUDA events around every launch, in a separate pass.  The card's name and power limit are
read in the same run.

    python scripts/bench_albert_text.py [--shapes albert_chinese_tiny,...] [--sentences 1024] [--ref-sentences 64]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_llm_text import card, packed_batches, sentence_lengths  # noqa: E402

from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.extract import albert_text as A  # noqa: E402


def reference_loop(m, ids, dev):
    with torch.no_grad():
        def fwd(x):
            hs = m(torch.from_numpy(x)[None].to(dev), output_hidden_states=True).hidden_states
            return torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0, 1:-1].cpu().numpy()
        for x in ids[:2]:
            fwd(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for x in ids:
            fwd(x)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def main():
    import transformers as tf
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(S.ALBERT_PUBLISHED_CFGS))
    ap.add_argument("--sentences", type=int, default=1024)
    ap.add_argument("--ref-sentences", type=int, default=64)
    ap.add_argument("--tokens", type=int, default=16384, help="tokens per packed pass")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    lens = [min(n, 512) for n in sentence_lengths(a.sentences, a.seed)]
    results = dict(card=name, power=power, lengths=dict(n=len(lens), mean=float(np.mean(lens)), total=int(sum(lens))))
    for shape in a.shapes.split(","):
        kw = S.ALBERT_PUBLISHED_CFGS[shape]
        rng = np.random.default_rng(a.seed + 1)
        ids = [np.concatenate([[2], rng.integers(10, kw["vocab_size"], n - 2), [3]]).astype(np.int64) for n in lens]
        cfg = tf.AlbertConfig(**kw)
        sd = S.albert_state_dict(kw, seed=a.seed + 7)
        m = tf.AlbertModel(cfg).eval()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
        m = m.to(dev)
        ref_ids = ids[:a.ref_sentences]
        ref_dt = reference_loop(m, ref_ids, dev)
        del m
        torch.cuda.empty_cache()
        d = A.AlbertDims(cfg)
        ops = A.CudaOps(A.default_precision(d.hidden), dev)
        net = A.AlbertNet({k: torch.from_numpy(v) for k, v in sd.items()}, ops, d)
        del sd

        def run():
            for batch in packed_batches(ids, a.tokens):
                net.forward(np.concatenate(batch), [len(x) for x in batch])
        with torch.no_grad():
            run()                                           # warm-up: every shape of the timed window
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                run()
            e1.record()
            torch.cuda.synchronize()
            dt = e0.elapsed_time(e1) / 1e3 / a.steps
            ops.timing = []
            run()
            torch.cuda.synchronize()
        shares = {}
        for klass, b, e in ops.timing:
            shares[klass] = shares.get(klass, 0.0) + b.elapsed_time(e)
        tot = sum(shares.values())
        r = dict(precision=ops.f16 and "f16" or "bf16x3", packed_sentences_per_s=len(ids) / dt,
                 packed_tokens_per_s=sum(lens) / dt, reference="HF fp32 batch 1",
                 reference_sentences_per_s=len(ref_ids) / ref_dt,
                 reference_tokens_per_s=sum(len(x) for x in ref_ids) / ref_dt,
                 speedup=(len(ids) / dt) / (len(ref_ids) / ref_dt), shares={k: v / tot for k, v in sorted(shares.items())})
        results[shape] = r
        print(f"{shape} ({r['precision']}): packed {r['packed_sentences_per_s']:.1f} sentences/s "
              f"({r['packed_tokens_per_s']:.0f} tokens/s); HF fp32 batch-1 loop {r['reference_sentences_per_s']:.2f} "
              f"sentences/s ({r['reference_tokens_per_s']:.0f} tokens/s); x{r['speedup']:.1f}")
        print(f"{shape}: time shares (per-launch events) " + ", ".join(f"{k} {v:.3f}" for k, v in r["shares"].items()))
        del net, ops
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
