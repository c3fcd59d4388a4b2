"""BIR-VAE measurements on one GPU (one process): fused train() images/s at B = 100 / 1024 / 8192, the MMD entry's time
against B with its exponentials (3 B^2) and FP32 operations counted from shapes, and the reference's torch
maximum_mean_discrepancy expression at the same B up to the largest that fits.  Alternated repeats; median and
spread.  Prints one JSON line; --out also writes it to a file.

python tools/bench_bir_vae.py [--repeats 5] [--out path]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "generative-models_b200")):
    sys.path.insert(0, p)

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32 (700 W)
MUFU_EX2_RATE = 132 * 16 * 1.98e9   # SFU ex2 per second at the boost clock: 16 per SM per clock (data-sheet clock)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def ref_mmd(z, x):
    """the reference's torch expression (src/bir_vae.py:190-211), with its prior sample already on z's device"""
    def k(a, b):
        n, m, d = a.size(0), b.size(0), a.size(1)
        ta, tb = a.unsqueeze(1).expand(n, m, d), b.unsqueeze(0).expand(n, m, d)
        return torch.exp(-torch.div(torch.mean(torch.pow(ta - tb, 2), dim=2), d))
    return k(x, x).sum() + k(z, z).sum() - 2 * k(x, z).sum()


def train_rate(B, steps):
    import bir_vae
    n = B * steps
    imgs = (torch.rand(n, 1, 28, 28, generator=torch.Generator().manual_seed(0)) < 0.13).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(n)), batch_size=B)
    val = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs[:B], torch.zeros(B)), batch_size=B)
    tr = bir_vae.BIRVAETrainer(bir_vae.BIRVAE(784, 400, 20), loader, val, val)
    tr.train(1)                                   # warm-up: engine, plans, resident dataset
    torch.cuda.synchronize()
    t = time.perf_counter()
    tr.train(1)
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import gm_b200
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": _card(), "train_images_per_s": {}, "mmd": []}
    import contextlib
    import io
    for B, steps in ((100, 200), (1024, 40), (8192, 8)):
        with contextlib.redirect_stdout(io.StringIO()):
            r = [train_rate(B, steps) for _ in range(a.repeats)]
        res["train_images_per_s"][B] = {"median": float(np.median(r)), "min": float(min(r)), "max": float(max(r))}
    Z = 20
    for B in (100, 1024, 4096, 8192, 16384, 32768):
        z, p = torch.randn(B, Z, device="cuda"), torch.randn(B, Z, device="cuda")
        ours, refs = [], []
        ref_ok = B * B * Z * 4 * 3 < 0.6 * torch.cuda.get_device_properties(0).total_memory
        iters = max(3, int(2e8 / (B * B)))
        for _ in range(a.repeats):                   # alternated: ours, reference, ours, ...
            ours.append(_events(lambda: gm_b200.mmd_gaussian(z, p, 1000.0), iters))
            if ref_ok:
                refs.append(_events(lambda: ref_mmd(z, p), max(1, iters // 10)))
        t = float(np.median(ours))
        exps = 3.0 * B * B
        flops = 3.0 * B * B * 3 * Z + 2.0 * B * B * 2 * Z    # 3 B^2 distances (Z FSUB + Z FFMA), 2 B^2 rows x Z product FFMAs
        row = {"B": B, "Z": Z, "ms_median": t * 1e3, "ms_min": min(ours) * 1e3, "ms_max": max(ours) * 1e3,
               "exp_per_s": exps / t, "fp32_flop_per_s": flops / t, "fp32_share_of_peak": flops / t / FP32_PEAK,
               "ex2_share_of_sfu": exps / t / MUFU_EX2_RATE,
               "reference_ms_median": float(np.median(refs)) * 1e3 if refs else None}
        res["mmd"].append(row)
        del z, p
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
