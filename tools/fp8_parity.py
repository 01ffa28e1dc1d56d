#!/usr/bin/env python
"""Loss-curve parity of the FP8 training mode against bf16 (BASELINE config #3 acceptance test).

Trains the same randomly initialised ResNet-50 (same seed, same cycling pool of synthetic batches, SGD momentum 0.9)
for --steps steps — bf16 operands (twice: the run-to-run gap of bf16 itself is the noise floor), then fp8 operands (e4m3
activations / weights, e5m2 gradients for the forward and data-gradient convolutions) — and compares the loss
trajectories: over the last 30 % of the run the fp8 curve must stay within max(--tol, 2 x noise floor) of a bf16 curve
(running means; the chaotic transient before that only has a blow-up guard), the final-window means must agree within --tol / 2,
and both must actually learn.
Each arm runs in its own process (clean kernel autotune / fp8 state).  Prints a markdown table
(and writes the curves as JSON with --json PATH).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def arm(precision, steps, batch, model, graph):
    import torch

    from distributeddeeplearning_b200.data import fixed_synthetic_batch
    from distributeddeeplearning_b200.ops import fp8
    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession

    dist.init()
    if precision == "fp8":
        fp8.enable(True)
    s = BenchmarkSession(model, batch, True, lr=0.01, momentum=0.9, seed=3)
    # 64 distinct batches (2,048 images, seen ~3 times in 200 steps): the loss falls steadily without collapsing to
    # ~0, where relative differences stop meaning anything
    pool = [fixed_synthetic_batch(batch, 224, 1000, s.device, seed=100 + i) for i in range(64)]
    losses = []
    for i in range(steps):
        if graph and i == 8:
            assert s.enable_graph(warmup=1), "graph capture failed"
        x, y = pool[i % len(pool)]
        l = s.step(x, y)
        losses.append(l.detach().clone())
    torch.cuda.synchronize()
    out = {"precision": precision, "losses": [float(v) for v in losses], "fp8_launches": fp8.launches(), "graph": bool(graph)}
    print("ARM " + json.dumps(out), flush=True)


def judge(b, b2, f, tol):
    """The acceptance rule, on three loss curves (bf16, bf16 again with the same seed, fp8).  Last 30 % of the run: the
    fp8 running mean stays within max(tol, 2 x what the two bf16 runs differ by) of the nearer bf16 run; before that (the
    loss overshoots to ~8.5 and comes back; two bf16 runs differ by 1-10 % there): only a blow-up guard at 2.5 x tol;
    final window: means within tol / 2 (or twice the bf16 spread); and both precisions must have learned."""
    n = len(b)
    win = max(10, n // 10)
    mean = lambda v: sum(v) / len(v)
    sm = lambda v: [mean(v[max(0, i - win + 1): i + 1]) for i in range(len(v))]     # batches differ in difficulty

    def curve_gaps(u, v):
        g = [abs(x - y) / x for x, y in zip(sm(u), sm(v))]
        cut = (7 * n) // 10                   # the transient (and every running-mean window touching it) is over by here
        return max(g[win:cut]), max(g[cut:])

    noise_early, noise = curve_gaps(b, b2)
    cand = [curve_gaps(b, f), curve_gaps(b2, f)]             # distance to the nearer of the two bf16 runs
    gap_early, gap = min(c[0] for c in cand), min(c[1] for c in cand)
    tail_b, tail_f = 0.5 * (mean(b[-win:]) + mean(b2[-win:])), mean(f[-win:])
    tail_noise = abs(mean(b[-win:]) - mean(b2[-win:])) / tail_b
    learned = tail_b < 0.97 * mean(b[:win]) and tail_f < 0.97 * mean(f[:win])
    ok = gap < max(tol, 2.0 * noise) and gap_early < max(2.5 * tol, 2.0 * noise_early) \
        and abs(tail_b - tail_f) / tail_b < max(0.5 * tol, 2.0 * tail_noise) and learned
    return {"ok": ok, "win": win, "gap": gap, "gap_early": gap_early, "noise": noise, "noise_early": noise_early,
            "tail_bf16": tail_b, "tail_fp8": tail_f, "tail_noise": tail_noise, "learned": learned}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--tol", type=float, default=0.08, help="allowed relative gap between the curves")
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--arm", default=None)
    ap.add_argument("--json", default=None, help="also write the curves and the verdict to this file")
    ap.add_argument("--fp8-mode", default="fp8", choices=["fp8"], help="which 8-bit mode to compare with bf16")
    a = ap.parse_args()
    if a.arm:
        return arm(a.arm, a.steps, a.batch, a.model, a.graph)
    res = {}
    # bf16 runs TWICE: the bf16 step is not bit-reproducible (atomics in the statistics / weight-gradient reductions:
    # a bf16 step is not bit-reproducible) and the first ~120 steps of this recipe are a chaotic transient, so two bf16 runs
    # of the same seed already differ by several per cent there.  That run-to-run gap is the noise floor the fp8 curve
    # is judged against.
    for p in ("bf16", "bf16_repeat", "fp8"):
        prec = a.fp8_mode if p == "fp8" else "bf16"
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", prec, "--steps", str(a.steps), "--batch",
                            str(a.batch), "--model", a.model, "--graph", str(a.graph)], capture_output=True, text=True,
                           timeout=1500)
        line = [l for l in r.stdout.splitlines() if l.startswith("ARM ")]
        if r.returncode != 0 or not line:
            print(r.stdout[-2000:], r.stderr[-3000:])
            return 1
        res[p] = json.loads(line[-1][4:])
    b, b2, f = res["bf16"]["losses"], res["bf16_repeat"]["losses"], res["fp8"]["losses"]
    n = len(b)
    v = judge(b, b2, f, a.tol)
    win, gap, gap_early, noise, noise_early = v["win"], v["gap"], v["gap_early"], v["noise"], v["noise_early"]
    tail_b, tail_f, tail_noise, learned = v["tail_bf16"], v["tail_fp8"], v["tail_noise"], v["learned"]
    ok = v["ok"] and res["fp8"]["fp8_launches"]["fwd"] > 0 and res["fp8"]["fp8_launches"]["dgrad"] > 0
    print(f"| step | bf16 loss | bf16 loss (same seed, second run) | fp8 loss |\n|---|---|---|---|")
    for i in list(range(0, n, max(1, n // 10))) + [n - 1]:
        print(f"| {i} | {b[i]:.4f} | {b2[i]:.4f} | {f[i]:.4f} |")
    print(f"\nmax relative gap of the {win}-step running means, fp8 vs the nearer bf16 run: last 30 % {gap:.4f} (bf16 vs bf16: "
          f"{noise:.4f}), before that {gap_early:.4f} (bf16 vs bf16: {noise_early:.4f}); last-{win}-step means: bf16 {tail_b:.4f} "
          f"(two runs differ by {tail_noise:.4f}), fp8 {tail_f:.4f}; "
          f"fp8 launches per run: {res['fp8']['fp8_launches']}; learned={learned}")
    print("FP8 PARITY:", "ok" if ok else "FAIL")
    if a.json:
        json.dump({"ok": ok, "gap": gap, "gap_early": gap_early, "noise_floor": noise, "noise_floor_early": noise_early,
                   "tail_bf16": tail_b, "tail_fp8": tail_f, "arms": res}, open(a.json, "w"))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
