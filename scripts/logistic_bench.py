"""Times LogisticRegression's device passes on the feature matrix in HBM — one loss / gradient evaluation
(lo_lr_loss_grad), transform and evaluate (lo_lr_predict) — and a whole fit, against a torch composition of one
evaluation on the same device (``x.double() @ W.T``, log-softmax or logsigmoid, ``X.T @ multipliers``), alternated in one
process, and checks that the two agree.  Prints the card and its power limit beside the figures.  Kernel time = the
call's kernels between CUDA events (lo_host_timing.kernel_ms); call time = CUDA events around the whole Python call.
Algorithmic bytes: loss / gradient and evaluate read n (4k + 4); transform reads n 4k and writes n 8 (C' + 1) with
C' = 2 when binomial.  Workloads: 10 M x 20 f32 binomial (Titanic-wide) and 100 M x 32 f32 with C = 10 (DESIGN.md
§3.6.3)."""
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from learningorchestra_b200.classifier import LogisticRegression  # noqa: E402
from learningorchestra_b200.engine import AssembledRows, Engine  # noqa: E402

PEAK = 3.35e12


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms))


def run(eng, n, k, nclasses, reps, fit_iters):
    g = torch.Generator(device="cuda").manual_seed(n + k)
    x = torch.randn((n, k), device="cuda", generator=g, dtype=torch.float32)
    w_true = torch.randn((nclasses, k), device="cuda", generator=g, dtype=torch.float32) * 0.3
    noise = -torch.log(-torch.log(torch.rand((n, nclasses), device="cuda", generator=g)))
    y = (x @ w_true.T + noise).argmax(1).to(torch.float32)
    del noise
    xt = eng.wrap("f32", n * k, 1, x.data_ptr(), n * k * 4, keepalive=x)
    yt = eng.wrap("f32", n, 1, y.data_ptr(), n * 4, keepalive=y)
    part = AssembledRows(xt, yt, None, k, n)
    multinomial = nclasses > 2
    nc = nclasses if multinomial else 1
    rng = np.random.default_rng(1)
    beta, b = rng.normal(size=(nc, k)) * 0.1, rng.normal(size=nc) * 0.1
    beta_t, b_t = torch.tensor(beta, device="cuda"), torch.tensor(b, device="cuda")
    yl = y.long()

    def t_loss_grad():
        m = x.double() @ beta_t.T + b_t
        if multinomial:
            logp = torch.log_softmax(m, 1)
            loss = -logp.gather(1, yl[:, None]).sum()
            mult = logp.exp()
            mult[torch.arange(n, device="cuda"), yl] -= 1.0
        else:
            yd = y.double()
            loss = -(yd * torch.nn.functional.logsigmoid(m[:, 0]) + (1 - yd) * torch.nn.functional.logsigmoid(-m[:, 0])).sum()
            mult = (torch.sigmoid(m[:, 0]) - yd)[:, None]
        return loss, x.double().T @ mult, mult.sum(0)

    loss, grad, gb = eng.lr_loss_grad(part, beta, b, multinomial)
    tl, tg, tb = t_loss_grad()
    agree = {"loss_rel": abs(loss - float(tl)) / abs(loss),
             "grad_max_rel": float(np.max(np.abs(grad - tg.T.cpu().numpy())) / np.max(np.abs(grad)))}
    res = {"n": n, "k": k, "C": nclasses, "agreement_with_torch": agree}
    kernel_ms = []

    def timing():
        tm = {}
        kernel_ms.append(tm)
        return tm

    labels = np.arange(nclasses, dtype=np.float64)
    nout = nclasses if multinomial else 2
    for name, ours, theirs, nbytes in (
            ("loss_grad", lambda: eng.lr_loss_grad(part, beta, b, multinomial, timing=timing()), t_loss_grad,
             n * (4 * k + 4)),
            ("transform", lambda: eng.lr_predict(part, beta, b, multinomial, timing=timing()).free(), None,
             n * 4 * k + n * 8 * (nout + 1)),
            ("evaluate", lambda: eng.lr_predict(part, beta, b, multinomial, labels=labels, timing=timing()), None,
             n * (4 * k + 4))):
        a, tb_ = [], []
        kernel_ms.clear()
        for _ in range(3):                     # alternate the two in one process
            a.append(timed(ours, reps))
            if theirs is not None:
                tb_.append(timed(theirs, reps))
        ms, kms = min(a), float(np.median([t["kernel_ms"] for t in kernel_ms]))
        res[name] = {"kernel_ms": round(kms, 3), "call_ms": round(ms, 3), "bytes": nbytes,
                     "kernel_share_of_3.35TBps_peak": round(nbytes / (kms * 1e-3) / PEAK, 3),
                     "call_share_of_3.35TBps_peak": round(nbytes / (ms * 1e-3) / PEAK, 3)}
        if tb_:
            res[name]["torch_ms"] = round(min(tb_), 3)
    feats = SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=eng)), _parts=[part],
                            fields=[f"f{j}" for j in range(k)], label="y", row_ids=np.arange(n), devices=[0])
    LogisticRegression(max_iter=2).fit(feats)                 # warm the fit's shapes
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m = LogisticRegression(max_iter=fit_iters).fit(feats)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    evals = len(m.objective_history) - 1
    res["fit"] = {"max_iter": fit_iters, "iterations": m.iterations, "seconds": round(wall, 3),
                  "ms_per_iteration": round(1e3 * wall / max(1, m.iterations), 3), "final_objective": m.objective_history[-1],
                  "states": evals + 1}
    return res


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    eng = Engine(0)
    results = [run(eng, 10_000_000, 20, 2, reps, 100), run(eng, 100_000_000, 32, 10, reps, 100)]
    print(json.dumps({"gpu": q, "results": results}))


if __name__ == "__main__":
    main()
