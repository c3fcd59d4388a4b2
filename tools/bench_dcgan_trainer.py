"""What the host batch costs the conv trainers' train(), and what the device-resident 8-bit pool (device_dataset) saves.

    python tools/bench_dcgan_trainer.py [--batch 1024] [--images 16384] [--rounds 3]

One GPU, one process.  DCGANTrainer (NSGAN) and DCVAETrainer at hidden 64, z 100 train on a host DataLoader(TensorDataset)
of N k/255 images (shuffle=True, batch B), the data the README's "more complex datasets" case implies.  Each trainer runs
train(num_epochs=1) with device_dataset off and on, alternated for --rounds rounds after one untimed call each way; the
wall clock around train() ends in a device synchronise.  The VAE's validation set is one batch of the same images, so its
epoch time is the training loop plus one evaluation batch.  Beside that:
  - the engine-only step (d_grad + apply + g_grad + apply; vae_grad + apply) on a resident batch, CUDA events per step, as
    tools/bench_dcgan.py times it;
  - the host path's batch alone: process_batch + stage_images, ending in a synchronise (median of 5);
  - gm_stage_pool_rows alone: CUDA events around --launches launches at B, as bytes moved (the codes read once, the bf16
    rows written) per second against the H100 SXM's 3.35 TB/s;
  - the one-off packing of the pool (DevicePool.from_loader);
  - a user-written loss: DCGANTrainer subclassed with the reference's NS train_D / train_G in torch (src/ns_gan.py:172-216),
    so train() runs the reference loop through the autograd nodes, against the fused DCGANTrainer.train on the same host
    loader, alternated for --rounds rounds, with the bytes the engine holds per D and per G call slot;
  - stage_images before (the torch expression it replaced) and after gm_image_to_rows: CUDA events around --launches calls
    at B on a device-resident fp32 batch.
Prints one JSON line with the device name and power limit read in the same run.  Writes nothing but stdout.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "generative-models_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_PEAK = 3.35e12                           # bytes/s, NVIDIA's H100 SXM data sheet


def _median(v):
    return sorted(v)[len(v) // 2]


def _event_ms(fn, count):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(count):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--images", type=int, default=16384)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    from torch.utils.data import DataLoader, TensorDataset
    import gm_b200
    import dc_gan
    import dc_vae
    from bench_dcgan import power_limit
    from gm_b200.dcgan import DevicePool
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcgan_trainer.py measures on a CUDA device; there is none")
    dev = torch.cuda.current_device()
    B, N = a.batch, a.images
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (N, 3, 64, 64), generator=g, dtype=torch.uint8).float().div_(255)
    loader = DataLoader(TensorDataset(images, torch.zeros(N)), batch_size=B, shuffle=True)
    val = DataLoader(TensorDataset(images[:B].clone(), torch.zeros(B)), batch_size=B, shuffle=False)
    torch.manual_seed(1)
    trainers = {"gan": dc_gan.DCGANTrainer(dc_gan.DCGAN(hidden_dim=64, z_dim=100), loader, val, val),
                "vae": dc_vae.DCVAETrainer(dc_vae.DCVAE(hidden_dim=64, z_dim=100), loader, val, val)}

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pool = DevicePool.from_loader(loader, 3)
    torch.cuda.synchronize()
    pack_s = time.perf_counter() - t0
    assert pool is not None, "the benchmark's loader must be eligible for the pool"
    for tr in trainers.values():
        tr._pool = pool                                              # reused by train() (same tensor and batching)

    def train(tr, on):
        tr.device_dataset = on
        torch.cuda.synchronize()
        t = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            tr.train(num_epochs=1)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit(dev), "batch": B, "images": N, "rounds": a.rounds,
           "hidden_dim": 64, "z_dim": 100, "pack_s": round(pack_s, 3), "pool_bytes": pool.codes.numel()}
    for name, tr in trainers.items():
        train(tr, False)
        train(tr, True)
        wall = {False: [], True: []}
        for _ in range(a.rounds):
            for on in (False, True):
                wall[on].append(train(tr, on))
        assert tr._pool is pool
        eng = tr._engine
        x = eng.stage_pool(pool, B, 5, 0).clone()
        hp = gm_b200.AdamHP.make(2e-4)
        if name == "gan":
            def step(s):
                eng.d_grad(x, B, seed=1000, step=s)
                eng.apply(1, hp)
                eng.g_grad(B, seed=1000, step=s)
                eng.apply(0, hp)
        else:
            def step(s):
                eng.vae_grad(x, B, seed=1000, step=s)
                eng.apply(hp)
        for s in range(a.warmup):
            step(s)
        torch.cuda.synchronize()
        eng_ms = _median([_event_ms(lambda i, s=s: step(100 + s), 1) for s in range(a.steps)])
        host = []
        for _ in range(5):
            torch.cuda.synchronize()
            t = time.perf_counter()
            eng.stage_images(tr.process_batch(loader) if name == "gan" else tr._images(next(iter(loader))))
            torch.cuda.synchronize()
            host.append((time.perf_counter() - t) * 1e3)
        off, on = _median(wall[False]), _median(wall[True])
        out[name] = {"off_s": [round(v, 4) for v in wall[False]], "on_s": [round(v, 4) for v in wall[True]],
                     "off_images_per_s": round(N / off, 1), "on_images_per_s": round(N / on, 1), "on_over_off": round(off / on, 3),
                     "engine_step_ms": round(eng_ms, 3), "engine_images_per_s": round(B / eng_ms * 1e3, 1),
                     "steps_per_epoch": len(loader), "host_batch_ms": round(_median(host), 2)}
    # at B (a train step's batch: a launch this short is bounded by the host's enqueue rate as much as by the kernel) and at
    # the whole pool (one long launch, the kernel's own rate)
    eng = trainers["gan"]._engine
    out["stage_pool_rows"] = []
    for rows in (B, N):
        for i in range(10):
            eng.stage_pool(pool, rows, 7, i)
        torch.cuda.synchronize()
        ms = _event_ms(lambda i: eng.stage_pool(pool, rows, 7, 10 + i), a.launches)
        moved = rows * pool.row_vals * 3 + 512                        # codes read, bf16 rows written, the table
        out["stage_pool_rows"].append({"rows": rows, "launches": a.launches, "us": round(ms * 1e3, 2), "bytes": moved,
                                       "tb_per_s": round(moved / (ms * 1e-3) / 1e12, 3),
                                       "of_hbm_peak": round(moved / (ms * 1e-3) / HBM_PEAK, 3)})
    out["custom_loss"] = custom_loss_leg(a, loader, B, N)
    print(json.dumps(out))


def custom_loss_leg(a, loader, B, N):
    import torch
    import dc_gan

    class NSOverride(dc_gan.DCGANTrainer):
        """the reference's NS losses (src/ns_gan.py:172-216) as a user override"""

        def train_D(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            G_output = self.model.G(noise)
            DX_score, DG_score = self.model.D(images), self.model.D(G_output)
            return torch.sum(-torch.mean(torch.log(DX_score + 1e-8) + torch.log(1 - DG_score + 1e-8)))

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            return -torch.mean(torch.log(self.model.D(self.model.G(noise)) + 1e-8))

    torch.manual_seed(2)
    trainers = {"fused": dc_gan.DCGANTrainer(dc_gan.DCGAN(hidden_dim=64, z_dim=100), loader, loader, loader),
                "custom": NSOverride(dc_gan.DCGAN(hidden_dim=64, z_dim=100), loader, loader, loader)}
    assert trainers["custom"]._has_custom_step() and not trainers["fused"]._has_custom_step()

    def train(tr):
        torch.cuda.synchronize()
        t = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            tr.train(num_epochs=1)
        torch.cuda.synchronize()
        return time.perf_counter() - t
    for tr in trainers.values():
        train(tr)
    wall = {k: [] for k in trainers}
    for _ in range(a.rounds):
        for k, tr in trainers.items():
            wall[k].append(train(tr))
    eng = trainers["custom"]._engine
    slot_bytes = {kind: sum(t.numel() * t.element_size() for key, t in eng._bufs.items() if key.startswith(pfx))
                  for kind, pfx in (("d_slot", "cd0"), ("g_slot", "cg0"), ("d_backward_shared", "cdb"))}
    out = {k: {"s": [round(v, 4) for v in w], "images_per_s": round(N / _median(w), 1)} for k, w in wall.items()}
    out["custom_over_fused_time"] = round(_median(wall["custom"]) / _median(wall["fused"]), 3)
    out["bytes"] = slot_bytes
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(B, 3 * 4096, device="cuda", generator=g)
    legs = {"torch_expression": lambda i: x.view(B, 3, 64, 64).permute(0, 2, 3, 1).to(torch.bfloat16).contiguous(),
            "gm_image_to_rows": lambda i: eng.stage_images(x)}
    for fn in legs.values():
        for i in range(10):
            fn(i)
    times = {k: [] for k in legs}
    for _ in range(3):
        for k, fn in legs.items():
            times[k].append(_event_ms(fn, a.launches))
    moved = B * 4096 * 3 * (4 + 2)                                    # fp32 read, bf16 written
    out["stage_images"] = {k: {"us": round(_median(v) * 1e3, 2), "tb_per_s": round(moved / (_median(v) * 1e-3) / 1e12, 3)}
                           for k, v in times.items()}
    out["stage_images"]["bytes"] = moved
    return out


if __name__ == "__main__":
    main()
