"""Bayesian GAN measurements on one GPU (one process), 784/400/20, J generator samples of B rows each:
- the fused Bayes step (d_grad + SGHMC of D, then g_grad + SGHMC of every generator sample, on a resident 1-bit pool with
  the in-kernel sampler and noise, as BayesGANTrainer.train() runs it), CUDA events;
- the fused NSGAN step (d_grad + Adam, g_grad + Adam, lazy gradients, as NSGANTrainer.train() runs it) at B rows,
  alternated with it, and their ratio;
- a torch-eager fp32 Bayesian GAN step (J nn.Sequential generators, one discriminator, SGHMC as torch ops) at the same
  shape as the baseline.
Both at J = 10, B = 8192 and at J = 10, B = 100 (the reference's batch), where the per-sample GEMM launches dominate.
Median, min and max over the repeats.  Prints one JSON line with the card's name and power limit; --out also writes it.

python tools/bench_bayes_gan.py [--samples 10] [--repeats 5] [--out path]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "generative-models_b200")):
    sys.path.insert(0, p)

X, H, Z = 784, 400, 20
N_POOL = 60000


def _card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def _stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def _timed(step, iters):
    step(0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for k in range(iters):
        step(k)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _bayes_ms(eng, bits, B, iters):
    import gm_b200
    hp = gm_b200.SghmcHP(2e-4, 0.1, 1.0, float(N_POOL))
    eng.set_sampler(N_POOL, 1)

    def step(k):
        eng.d_grad(bits, fmt="bits", batch=B, seed=1, step=k)
        eng.apply(1, hp, seed=1, step=k)
        eng.g_grad(B, seed=1, step=k)
        eng.apply(0, hp, seed=1, step=k)
    return _timed(step, iters)


def _ns_ms(eng, bits, B, iters):
    import gm_b200
    hp = gm_b200.AdamHP.make(2e-4)
    eng.set_lazy_grads(True)
    eng.set_sampler(N_POOL, 1)

    def step(k):
        eng.d_grad(bits, fmt="bits", batch=B, seed=1, step=k)
        eng.apply(1, hp)
        eng.g_grad(B, seed=1, step=k)
        eng.apply(0, hp)
    try:
        return _timed(step, iters)
    finally:
        eng.set_lazy_grads(False)


def _eager_ms(J, B, iters):
    Gs = [nn.Sequential(nn.Linear(Z, H), nn.ReLU(), nn.Linear(H, X), nn.Sigmoid()).cuda() for _ in range(J)]
    Dn = nn.Sequential(nn.Linear(X, H), nn.ReLU(), nn.Linear(H, 1), nn.Sigmoid()).cuda()
    x = (torch.rand(B, X, device="cuda") < 0.13).float()
    lr, alpha, N = 2e-4, 0.1, float(N_POOL)
    mom = {p: torch.zeros_like(p) for m in Gs + [Dn] for p in m.parameters()}

    @torch.no_grad()
    def sghmc(params):
        for p in params:
            v = mom[p]
            v.mul_(1 - alpha).add_(p.grad + p / N, alpha=-lr).add_(torch.randn_like(p), alpha=(2 * alpha * lr / N) ** 0.5)
            p.add_(v)

    def step(_):
        for m in Gs + [Dn]:
            m.zero_grad()
        with torch.no_grad():
            fake = torch.cat([g(torch.randn(B, Z, device="cuda")) for g in Gs])
        (-torch.mean(torch.log(Dn(x) + 1e-8)) - torch.mean(torch.log(1 - Dn(fake) + 1e-8))).backward()
        sghmc(Dn.parameters())
        Dn.zero_grad()
        sum(-torch.mean(torch.log(Dn(g(torch.randn(B, Z, device="cuda"))) + 1e-8)) for g in Gs).backward()
        sghmc([p for g in Gs for p in g.parameters()])
    return _timed(step, iters)


def _case(J, B, repeats, bits):
    import gm_b200
    be = gm_b200.BayesGanEngine(X, H, Z, num_g=J, max_batch=B)
    ne = gm_b200.GanEngine(X, H, Z, max_batch=B, variant="ns")
    torch.manual_seed(0)
    for net, eng in ((0, be), (1, be), (0, ne), (1, ne)):
        for s in range(J if eng is be and net == 0 else 1):
            w = [torch.randn(v.shape) * 0.03 for v in eng.views(net)]
            if eng is be:
                eng.load(net, w, sample=s)
            else:
                eng.load(net, w)
    iters = 10 if B > 1000 else 100
    sb, sn = [], []
    _bayes_ms(be, bits, B, 2)                       # warm-up: plans and modules
    _ns_ms(ne, bits, B, 2)
    for _ in range(repeats):                        # alternated: Bayes, NS, Bayes, ...
        sb.append(_bayes_ms(be, bits, B, iters))
        sn.append(_ns_ms(ne, bits, B, iters))
    del be, ne
    torch.cuda.empty_cache()
    eager = [_eager_ms(J, B, 5 if B > 1000 else 20) for _ in range(max(2, repeats // 2))]
    return {"samples": J, "batch": B, "bayes_step_ms": _stats(sb), "ns_step_ms": _stats(sn),
            "bayes_over_ns_step_time": _stats([a / b for a, b in zip(sb, sn)]), "eager_bayes_step_ms": _stats(eager),
            "eager_over_fused_bayes": float(np.median(eager) / np.median(sb))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gm_b200.gan_api import DeviceDataset
    g = torch.Generator(device="cuda").manual_seed(0)
    bits = DeviceDataset((torch.rand(N_POOL, X, device="cuda", generator=g) < 0.13).float(), 8192).bits
    res = {"card": _card(), "shape": [X, H, Z],
           "cases": [_case(a.samples, 8192, a.repeats, bits), _case(a.samples, 100, a.repeats, bits)]}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
