#!/usr/bin/env python
"""Golden fixture tests/golden/bir_vae.npz: the UNMODIFIED reference src/bir_vae.py run on the CPU with the seeded
inputs of inputs.py (the same set-up as make_golden.py's vae case, whose helpers it uses).  Stored: the numpy eps draws
(np.random.normal in reparameterize) and the torch prior draws (torch.randn in maximum_mean_discrepancy) in call order,
the per-step mse / mmd losses of the reference's own train(), the step-1 losses and gradients of compute_batch +
backward, and the final weights.  Initial weights come from gm_init_weights(BIR_SHAPES, 4322).

Usage:  python tests/golden/make_golden_bir_vae.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
from inputs import B, X, H, Z, STEPS, gm_init_weights, gm_images  # noqa: E402

BIR_SHAPES = [("encoder.linear", (H, X)), ("encoder.mu", (Z, H)), ("decoder.linear", (H, Z)), ("decoder.recon", (X, H))]
SEED = 4322


class NormalRecorder:
    """record every np.random.normal result (call order)"""

    def __init__(self):
        self.draws = []
        self._normal = np.random.normal

    def __enter__(self):
        def normal(*a, **k):
            r = self._normal(*a, **k)
            self.draws.append(np.asarray(r, dtype=np.float32))
            return r
        np.random.normal = normal
        return self

    def __exit__(self, *exc):
        np.random.normal = self._normal


def main():
    mod = mg.import_ref("bir_vae")
    torch.set_num_threads(1)
    weights = gm_init_weights(BIR_SHAPES, seed=SEED)
    imgs = gm_images(B)
    images4d = torch.from_numpy(imgs.copy()).view(B, 1, 28, 28)
    it = [(images4d, torch.zeros(B, dtype=torch.long))] * STEPS
    out = {"images_bits": np.packbits(imgs.astype(np.uint8), axis=None)}

    model = mod.BIRVAE(X, H, Z, I=13.3)
    mg.load_weights(model, weights)
    trainer = mod.BIRVAETrainer(model, it, it[:1], it[:1], viz=False)
    torch.manual_seed(20240924)
    np.random.seed(20240924)
    with mg.DrawRecorder() as rec, NormalRecorder() as nrec:
        trainer.train(num_epochs=1, lr=1e-3, weight_decay=1e-5)
    out["recon_loss"] = np.asarray(trainer.recon_loss, dtype=np.float64)
    out["mmd_loss"] = np.asarray(trainer.mmd_loss, dtype=np.float64)
    out["eps"] = np.stack(nrec.draws)                        # STEPS train draws + 1 validation draw
    mg.pack_draws(rec.draws, out)
    for name, p in model.state_dict().items():
        mg.summarise("final_" + name, p.numpy(), out)

    model2 = mod.BIRVAE(X, H, Z, I=13.3)
    mg.load_weights(model2, weights)
    tr2 = mod.BIRVAETrainer(model2, it, it[:1], it[:1], viz=False)
    torch.manual_seed(20240924)
    np.random.seed(20240924)
    with mg.DrawRecorder() as rec2, NormalRecorder() as nrec2:
        mse, mmd = tr2.compute_batch(it[0])
        (mse + mmd).backward()
    out["step1_mse"] = np.float64(mse.item())
    out["step1_mmd"] = np.float64(mmd.item())
    out["step1_eps"] = nrec2.draws[0]
    out["step1_prior"] = rec2.draws[0][1]
    for name, p in model2.named_parameters():
        mg.summarise("step1_grad_" + name, p.grad.numpy(), out)
    np.savez_compressed(os.path.join(HERE, "bir_vae.npz"), **out)
    print("bir_vae mse %s mmd %s" % (np.round(out["recon_loss"], 4), np.round(out["mmd_loss"], 5)))


if __name__ == "__main__":
    main()
