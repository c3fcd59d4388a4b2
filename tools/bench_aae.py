"""Adversarial autoencoder measurements on one GPU (one process), at B = 131072 and 784/400/20:
- the fused AAE step (recon_grad + apply, d_grad + apply_d, g_grad + apply_g on a resident 1-bit pool, with the in-kernel
  sampler and prior draw, as AAETrainer.train() runs it), CUDA events;
- the fused VAE step (grad + apply, as VAETrainer.train() runs it) at the same shape, alternated with it, and their ratio;
- a torch-eager AAE (nn.Linear layers, fp32, three torch.optim.Adam) step on the same GPU as the baseline.
Median, min and max over the repeats.  Prints one JSON line with the card's name and power limit; --out also writes it.

python tools/bench_aae.py [--batch 131072] [--steps 4] [--repeats 5] [--out path]"""
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


def _aae_ms(eng, bits, n, steps, B, iters=10):
    import gm_b200
    hpR, hpD, hpG = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5), gm_b200.AdamHP.make(2e-4), gm_b200.AdamHP.make(2e-4)
    eng.set_lazy_grads(True)
    eng.set_sampler(n, steps, 1, batch_size=B)

    def step(k):
        eng.recon_grad(bits, fmt="bits", batch=B, step=k)
        eng.apply(hpR)
        eng.d_grad(B, seed=1, step=k)
        eng.apply_d(hpD)
        eng.g_grad(B)
        eng.apply_g(hpG)
    try:
        return _timed(step, iters)
    finally:
        eng.set_lazy_grads(False)
        eng.set_sampler(0, 0, 0)


def _vae_ms(eng, bits, n, steps, B, iters=10):
    import gm_b200
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    eng.set_lazy_grads(True)
    eng.set_sampler(n, steps, 1, batch_size=B)

    def step(k):
        eng.grad(bits, fmt="bits", batch=B, seed=1, step=k)
        eng.apply(hp)
    try:
        return _timed(step, iters)
    finally:
        eng.set_lazy_grads(False)
        eng.set_sampler(0, 0, 0)


def _eager_ms(B, iters=5):
    enc = nn.Sequential(nn.Linear(X, H), nn.ReLU(), nn.Linear(H, Z)).cuda()
    dec = nn.Sequential(nn.Linear(Z, H), nn.ReLU(), nn.Linear(H, X), nn.Sigmoid()).cuda()
    dis = nn.Sequential(nn.Linear(Z, H), nn.ReLU(), nn.Linear(H, 1), nn.Sigmoid()).cuda()
    oR = torch.optim.Adam(list(enc.parameters()) + list(dec.parameters()), lr=1e-3, weight_decay=1e-5)
    oD, oG = torch.optim.Adam(dis.parameters(), lr=2e-4), torch.optim.Adam(enc.parameters(), lr=2e-4)
    x = (torch.rand(B, X, device="cuda") < 0.13).float()

    def step(_):
        oR.zero_grad()
        ((x - dec(enc(x))) ** 2).sum().backward()
        oR.step()
        oD.zero_grad()
        zf = enc(x).detach()
        (-torch.mean(torch.log(dis(torch.randn(B, Z, device="cuda")) + 1e-8) + torch.log(1 - dis(zf) + 1e-8))).backward()
        oD.step()
        oG.zero_grad()
        (-torch.mean(torch.log(dis(enc(x)) + 1e-8))).backward()
        oG.step()
    return _timed(step, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--steps", type=int, default=4, help="batches per epoch of the resident pool")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import gm_b200
    from gm_b200.gan_api import DeviceDataset
    B, n = a.batch, a.batch * a.steps
    g = torch.Generator(device="cuda").manual_seed(0)
    bits = DeviceDataset((torch.rand(n, X, device="cuda", generator=g) < 0.13).float(), B).bits
    ae, ve = gm_b200.AaeEngine(X, H, Z, max_batch=B), gm_b200.VaeEngine(X, H, Z, max_batch=B)
    torch.manual_seed(0)
    ae.load({k: torch.randn(v.shape) * 0.03 for k, v in ae.views().items()})
    ve.load({k: torch.randn(v.shape) * 0.03 for k, v in ve.views().items()})
    sa, sv = [], []
    _aae_ms(ae, bits, n, a.steps, B, 2)                  # warm-up: plans and modules
    _vae_ms(ve, bits, n, a.steps, B, 2)
    for _ in range(a.repeats):                           # alternated: AAE, VAE, AAE, ...
        sa.append(_aae_ms(ae, bits, n, a.steps, B))
        sv.append(_vae_ms(ve, bits, n, a.steps, B))
    del ae, ve
    torch.cuda.empty_cache()
    eager = [_eager_ms(B) for _ in range(max(2, a.repeats // 2))]
    ratio = [x / v for x, v in zip(sa, sv)]
    res = {"card": _card(), "batch": B, "shape": [X, H, Z], "aae_step_ms": _stats(sa), "vae_step_ms": _stats(sv),
           "aae_over_vae_step_time": _stats(ratio), "eager_aae_step_ms": _stats(eager),
           "eager_over_fused_aae": float(np.median(eager) / np.median(sa)),
           "aae_images_per_s": B / (np.median(sa) * 1e-3), "eager_images_per_s": B / (np.median(eager) * 1e-3)}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
