"""Time the two regimes of the fit sweep (GradCore::sweep, csrc/grad_kernel.cuh) at the C2 benchmark's shapes, with CUDA
events, and print one JSON line with the card, its power limit and its SM clock:

  fit   rcmarl_grad over the whole steady-state buffer (3 000 time rows x 4 096 environments = 12.29 M rows) with the
        C2 job table of the full-batch local fits: 4 cooperative agents x (team-reward net on sa, targets = one column
        of r at stride 5; critic on s, TD targets at stride 1) = 8 jobs, as update_round launches it (fit_grad);
  mb    rcmarl_minibatch_fit of the malicious agent's three chains (critic_local / team reward / critic, targets at
        stride 1) over the same buffer: 10 epochs x 94 mini-batches of 32 time rows x 4 096 environments = 940 SGD steps
        (minibatch_sgd).

Inputs are seeded, so two builds see the same data.  RCMARL_LIB selects the library, so a parent build and a new build
can be run one after the other in the same session:

    RCMARL_LIB=/path/to/librcmarl.so python tools/prof_sweep.py [--reps 3] [--out DIR]

Besides the timings the line carries the SHA-256 of the fit's gradient sums and of the chains' weights after one call,
so that two builds can be compared bit for bit; --out also writes them as DIR/fit_sums.npy and DIR/mb_weights.npy.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
from rcmarl import ops, nets, _lib as L   # noqa: E402

NA, T, N = 5, 3000, 4096
EPOCHS, MB_TIMES, LR = 10, 32, 0.01


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, launches, reps):
    """median over reps of the mean time per launch (ms) of `launches` back-to-back launches"""
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / launches)
    return float(np.median(ts)), [float(t) for t in ts]


def sha(t):
    return hashlib.sha256(t.detach().cpu().numpy().tobytes()).hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fit-launches", type=int, default=20)
    ap.add_argument("--mb-calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    rows_n = T * N
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    sa = torch.randn(rows_n, 3 * NA, device=dev, generator=g)
    ns = torch.randn(rows_n, 2 * NA, device=dev, generator=g)
    r = torch.randn(rows_n, NA, device=dev, generator=g)
    tdt = torch.randn(4, rows_n, device=dev, generator=g)
    rs = np.random.RandomState(0)
    PC, PT = L.param_count(2 * NA, 1), L.param_count(3 * NA, 1)
    wc = [torch.as_tensor(nets.pack(nets.glorot_uniform(2 * NA, 1, rs))).to(dev) for _ in range(4)]
    wt = [torch.as_tensor(nets.pack(nets.glorot_uniform(3 * NA, 1, rs))).to(dev) for _ in range(4)]
    ws = ops.workspace()

    # ---- full-batch fit: the C2 job table (team-reward targets = r[:, i] at stride NA, critic targets at stride 1)
    sums = torch.zeros(8, PT + 1, device=dev)
    rows = ops.make_rows(sa, ns, r, NA)
    jobs = []
    for i in range(4):
        jobs.append(ops.grad_job(wt[i], r[:, i], sums[2 * i], L.IN_SA, target_stride=NA))
        jobs.append(ops.grad_job(wc[i], tdt[i], sums[2 * i + 1][:PC + 1], L.IN_S))
    jobs = ops.job_array(L.GradJob, jobs)
    fit = lambda: ops.grad(rows, jobs, L.LOSS_MSE, ws)   # noqa: E731
    for _ in range(3):
        fit()
    torch.cuda.synchronize()
    fit_sums = sums.clone()
    fit_ms, fit_all = timed(fit, args.fit_launches, args.reps)

    # ---- mini-batch chains of one malicious agent: critic_local (s), team reward (sa), critic (s), all at stride 1
    w0 = [wc[0], wt[1], wc[2]]
    kinds = [L.IN_S, L.IN_SA, L.IN_S]
    tgts = [tdt[0], tdt[1], tdt[2]]
    w = [x.clone() for x in w0]
    sums_mb = torch.zeros(3, PT + 1, device=dev)
    perms = torch.stack([torch.stack([torch.randperm(T, generator=torch.Generator().manual_seed(100 * c + e))
                                      for e in range(EPOCHS)]) for c in range(3)]).to(torch.int32).to(dev)
    gj, aj = [], []
    for c in range(3):
        n = PT if kinds[c] == L.IN_SA else PC
        gj.append(ops.grad_job(w[c], tgts[c], sums_mb[c][:n + 1], kinds[c], time_idx=perms[c]))
        aj.append(ops.sgd_job(w[c], w[c], sums_mb[c][:n + 1], n, LR))
    gj, aj = ops.job_array(L.GradJob, gj), ops.job_array(L.SgdJob, aj)
    mb_rows = ops.make_rows(sa, ns, r, NA, 0, 0, perms, N)
    cells = ops.MinibatchCells(L.MAX_JOBS, PT, dev)

    def mb():
        for x, x0 in zip(w, w0):
            x.copy_(x0)
        ops.minibatch_fit(mb_rows, gj, aj, EPOCHS, T, MB_TIMES, LR, cells)
    mb()
    torch.cuda.synchronize()
    mb_w = torch.cat([x.clone() for x in w])
    mb()
    torch.cuda.synchronize()
    mb_ms, mb_all = timed(mb, args.mb_calls, args.reps)
    steps = L.lib().rcmarl_minibatch_steps(EPOCHS, T, MB_TIMES)
    same_mb = bool(torch.equal(mb_w, torch.cat(w)))

    if args.out:
        os.makedirs(args.out, exist_ok=True)
        np.save(os.path.join(args.out, "fit_sums.npy"), fit_sums.cpu().numpy())
        np.save(os.path.join(args.out, "mb_weights.npy"), mb_w.cpu().numpy())
    print(json.dumps(dict(lib=L.LIB_PATH, card=card(), fit_rows=rows_n, fit_jobs=8, fit_ms_per_launch=fit_ms,
                          fit_ms_reps=fit_all, mb_steps=steps, mb_ms_per_call=mb_ms, mb_us_per_step=1e3 * mb_ms / steps,
                          mb_ms_reps=mb_all, fit_sums_sha=sha(fit_sums), mb_weights_sha=sha(mb_w),
                          mb_repeatable=same_mb)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
