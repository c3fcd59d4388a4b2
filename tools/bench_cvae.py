"""Conditional VAE measurements on one GPU (one process), at B = 131072 and 784/400/20 with C = 10:
- fused CVAETrainer.train() images/s (resident 1-bit images and int32 labels, in-kernel sampler and eps), and
  VAETrainer.train() at the same shape, alternated with it in the same call;
- the engine step alone (grad + apply on the resident pool, CUDA events) for both, alternated, and their ratio;
- a torch-eager CVAE (nn.Linear layers, fp32, torch.optim.Adam) step on the same GPU as the baseline.
Median, min and max over the repeats.  Prints one JSON line with the card's name and power limit; --out also writes it.

python tools/bench_cvae.py [--batch 131072] [--steps 4] [--repeats 5] [--out path]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "generative-models_b200")):
    sys.path.insert(0, p)

X, H, Z, K = 784, 400, 20, 10


def _card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def _stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def _trainers(B, steps):
    import cvae
    import vae
    n = B * steps
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = (torch.rand(n, 1, 28, 28, device="cuda", generator=g) < 0.13).float()
    labels = torch.randint(0, K, (n,), device="cuda", generator=g)
    ds = torch.utils.data.TensorDataset(imgs, labels)
    loader = torch.utils.data.DataLoader(ds, batch_size=B)
    val = [(imgs[:1024].cpu(), labels[:1024].cpu())]
    tc = cvae.CVAETrainer(cvae.CVAE(X, H, Z, K), loader, val, val)
    tv = vae.VAETrainer(vae.VAE(X, H, Z), loader, val, val)
    return tc, tv, n


def _train_rate(tr, n):
    torch.cuda.synchronize()
    t = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        tr.train(1)
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t)


def _step_ms(tr, steps, iters=10):
    """grad + apply of the trainer's engine on its resident pool, as train() runs them, timed with CUDA events"""
    import gm_b200
    res, eng = tr._resident, tr._engine
    B = min(res.batch_size, res.n)
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    labels = tr._resident_y[1] if hasattr(tr, "_resident_y") else None
    eng.set_lazy_grads(True)
    eng.set_sampler(res.n, steps, 1, batch_size=B)

    def step(k):
        if labels is None:
            eng.grad(res.bits, fmt="bits", batch=B, seed=1, step=k)
        else:
            eng.grad(res.bits, labels, fmt="bits", batch=B, seed=1, step=k)
        eng.apply(hp)
    try:
        step(0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for k in range(iters):
            step(k)
        b.record()
        b.synchronize()
    finally:
        eng.set_lazy_grads(False)
        eng.set_sampler(0, 0, 0)
    return a.elapsed_time(b) / iters


class EagerCVAE(nn.Module):
    def __init__(self):
        super().__init__()
        self.e1, self.mu, self.lv = nn.Linear(X + K, H), nn.Linear(H, Z), nn.Linear(H, Z)
        self.d1, self.d2 = nn.Linear(Z + K, H), nn.Linear(H, X)

    def forward(self, x, y):
        oh = F.one_hot(y, K).float()
        h = torch.relu(self.e1(torch.cat([x, oh], 1)))
        mu, lv = self.mu(h), self.lv(h)
        z = mu + torch.randn_like(mu) * torch.exp(lv / 2)
        return torch.sigmoid(self.d2(torch.relu(self.d1(torch.cat([z, oh], 1))))), mu, lv


def _eager_ms(B, iters=5):
    m = EagerCVAE().cuda()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-5)
    x = (torch.rand(B, X, device="cuda") < 0.13).float()
    y = torch.randint(0, K, (B,), device="cuda")

    def step():
        opt.zero_grad()
        out, mu, lv = m(x, y)
        loss = ((x - out) ** 2).sum() + torch.sum(0.5 * (mu ** 2 + torch.exp(lv) - lv - 1))
        loss.backward()
        opt.step()
    step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--steps", type=int, default=4, help="batches per train() epoch")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    B = a.batch
    tc, tv, n = _trainers(B, a.steps)
    for tr in (tc, tv):                                  # warm-up: engines, plans, resident dataset and labels
        _train_rate(tr, n)
    rc, rv, sc, sv = [], [], [], []
    for _ in range(a.repeats):                           # alternated: CVAE, VAE, CVAE, ...
        rc.append(_train_rate(tc, n))
        rv.append(_train_rate(tv, n))
        sc.append(_step_ms(tc, a.steps))
        sv.append(_step_ms(tv, a.steps))
    eager = [_eager_ms(B) for _ in range(max(2, a.repeats // 2))]
    ratio = [c / v for c, v in zip(sc, sv)]
    res = {"card": _card(), "batch": B, "shape": [X, H, Z, K],
           "cvae_train_images_per_s": _stats(rc), "vae_train_images_per_s": _stats(rv),
           "cvae_step_ms": _stats(sc), "vae_step_ms": _stats(sv), "cvae_over_vae_step_time": _stats(ratio),
           "eager_cvae_step_ms": _stats(eager), "cvae_images_per_s_from_step": B / (np.median(sc) * 1e-3),
           "eager_images_per_s": B / (np.median(eager) * 1e-3)}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
