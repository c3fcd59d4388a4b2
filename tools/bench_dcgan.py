"""Conv NSGAN, MMGAN, WGAN, LSGAN, f-GAN (Jensen-Shannon), RaNSGAN, Fisher GAN, WGAN-GP, DRAGAN, BEGAN and InfoGAN train
steps (D_steps = 1) and the conv VAE and autoencoder steps on one GPU, in one process.

    python tools/bench_dcgan.py [--batch 1024] [--steps 20] [--warmup 5]

Every engine runs the DCGAN of bench.py's dcgan workload (64x64x3, hidden 64, z 100) on that workload's image pool:
device-resident binarised synthetic images (each value 1 with probability 0.3), four batches cycled.  The legs run in two
groups (GROUPS: all thirteen engines at batch 1024 do not fit in 80 GB at once), each with its own NSGAN leg ("ns",
"ns_group2") that its over_ns ratios use.  Within a group the steps alternate (rounds of one step per variant, each timed
with its own CUDA events after the warm-up), so clock or thermal drift hits all alike.  Prints one JSON line: device name and power limit (read in the same run), and per variant the median step
time, images/s, library launches per step, the ratio to NSGAN and achieved TFLOP/s from FLOPs counted from the shapes
(bench.py's _dcgan_flop_per_img; the penalised critics of WGAN-GP and DRAGAN add one critic forward, one input-gradient
chain to the image, one tangent forward and one weight-gradient pass = 4 critic forwards; BEGAN's from its autoencoder's
shapes, began_flop_per_img; InfoGAN's from its G, D and Q shapes, info_flop_per_img; the VAE's from its encoder and
decoder shapes, vae_flop_per_img; the autoencoder's from the same with a z-wide head).  BEGAN's step includes began_control, and InfoGAN's the MI step and MI_optimizer's update
(q_grad + apply_mi), as their trainers run them after every G update.  The VAE step is vae_grad + apply (one Adam over
encoder and decoder, lr 1e-3, weight decay 1e-5, src/vae.py:139-142) on the same images; the autoencoder's is ae_grad +
apply with the same optimizer (src/ae.py:98-101) and the reference's code width z = 32 (src/ae.py:58).  WGAN's D Adam clamps
to [-0.01, 0.01] (src/w_gan.py:105).  Writes nothing but stdout.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "generative-models_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

# two groups of alternated legs, each with its own NSGAN leg: the thirteen engines at batch 1024 do not fit in 80 GB together
GROUPS = (("ns", "ra", "fisher", "wgp", "dra", "be", "info", "vae"), ("ns", "mm", "w", "ls", "f_jensen_shannon", "ae"))
LR = {"ns": 2e-4, "mm": 2e-4, "w": 5e-5, "ls": 1e-4, "f_jensen_shannon": 1e-4, "ra": 2e-4, "fisher": 1e-4, "wgp": 1e-4, "dra": 1e-4,
      "be": 1e-4, "info": 2e-4, "vae": 1e-3, "ae": 1e-3}   # the reference's defaults
AE_Z = 32                                                   # the autoencoder's code width (src/ae.py:58)


def critic_flop_per_img(hd=64, ch=3):
    dc = [hd, 2 * hd, 4 * hd, 8 * hd]
    d_l = [1024 * dc[0] * 16 * ch, 256 * dc[1] * 16 * dc[0], 64 * dc[2] * 16 * dc[1], 16 * dc[3] * 16 * dc[2], 16 * dc[3]]
    return 2.0 * sum(d_l)


def began_flop_per_img(hd=64, z=100, e=100, ch=3):
    """algorithmic FLOPs of one BEGAN step, counted like bench.py's _dcgan_flop_per_img: D step = G fwd + 2 autoencoder fwd +
    2 autoencoder bwd (weight grads everywhere, input grads down to the encoder's first layer); G step = G fwd + autoencoder
    fwd + its input-gradient chain down to the image + G bwd"""
    gc, dc = [8 * hd, 4 * hd, 2 * hd, hd, ch], [hd, 2 * hd, 4 * hd, 8 * hd]
    enc = [1024 * dc[0] * 16 * ch, 256 * dc[1] * 16 * dc[0], 64 * dc[2] * 16 * dc[1], 16 * dc[3] * 16 * dc[2], 16 * dc[3] * e]
    g_l = [z * 16 * gc[0], 16 * gc[0] * 16 * gc[1], 64 * gc[1] * 16 * gc[2], 256 * gc[2] * 16 * gc[3], 1024 * gc[3] * 16 * gc[4]]
    dec = [e * 16 * gc[0]] + g_l[1:]
    ae = sum(enc) + sum(dec)
    Gf, AEf = 2.0 * sum(g_l), 2.0 * ae
    ae_bwd = 2.0 * (2 * ae - enc[0])                 # wgrad everywhere + dgrad except into the image
    ae_dgrad = 2.0 * ae                              # G step: input-gradient chain only, down to the image
    g_bwd = 2.0 * (2 * sum(g_l) - g_l[0])
    return (Gf + 2 * AEf + 2 * ae_bwd) + (Gf + AEf + ae_dgrad + g_bwd)


def info_flop_per_img(hd=64, z=100, nd=10, nc=10, ch=3):
    """algorithmic FLOPs of one InfoGAN step, counted like bench.py's _dcgan_flop_per_img: the NSGAN D and G steps with G's
    input z + nd + nc wide, then the MI step = G fwd + Q fwd + Q bwd (weight grads everywhere, input grads down to the
    image) + G bwd"""
    from bench import _dcgan_flop_per_img
    gc, dc = [8 * hd, 4 * hd, 2 * hd, hd, ch], [hd, 2 * hd, 4 * hd, 8 * hd]
    q_l = [1024 * dc[0] * 16 * ch, 256 * dc[1] * 16 * dc[0], 64 * dc[2] * 16 * dc[1], 16 * dc[3] * 16 * dc[2], 16 * dc[3] * (nd + nc)]
    g_l = [(z + nd + nc) * 16 * gc[0], 16 * gc[0] * 16 * gc[1], 64 * gc[1] * 16 * gc[2], 256 * gc[2] * 16 * gc[3], 1024 * gc[3] * 16 * gc[4]]
    mi = 2.0 * sum(g_l) + 2.0 * sum(q_l) + 2.0 * (2 * sum(q_l)) + 2.0 * (2 * sum(g_l) - g_l[0])
    return _dcgan_flop_per_img(hd, z + nd + nc, ch) + mi


def vae_flop_per_img(hd=64, z=100, ch=3, heads=2):
    """algorithmic FLOPs of one VAE step, counted like bench.py's _dcgan_flop_per_img: encoder fwd (the D trunk with the
    heads x z-wide head) + decoder fwd (the generator) + decoder bwd (weight grads everywhere, input grads down to z) + encoder
    bwd (weight grads everywhere, no input gradient into the image).  heads=1: the autoencoder's step"""
    gc, dc = [8 * hd, 4 * hd, 2 * hd, hd, ch], [hd, 2 * hd, 4 * hd, 8 * hd]
    enc = [1024 * dc[0] * 16 * ch, 256 * dc[1] * 16 * dc[0], 64 * dc[2] * 16 * dc[1], 16 * dc[3] * 16 * dc[2], 16 * dc[3] * heads * z]
    dec = [z * 16 * gc[0], 16 * gc[0] * 16 * gc[1], 64 * gc[1] * 16 * gc[2], 256 * gc[2] * 16 * gc[3], 1024 * gc[3] * 16 * gc[4]]
    return 2.0 * sum(enc) + 2.0 * sum(dec) + 2.0 * (2 * sum(dec)) + 2.0 * (2 * sum(enc) - enc[0])


def power_limit(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def run_group(variants, a, pool):
    """one group of alternated legs (their engines are alive together); over_ns_images_per_s against the group's own NSGAN"""
    import torch
    import gm_b200
    from bench import _dcgan_flop_per_img
    B = a.batch
    engines = {v: gm_b200.DcganEngine(64, AE_Z if v == "ae" else 100, 3, variant=v) for v in variants}
    hps = {v: gm_b200.AdamHP.make(LR[v], weight_decay=1e-5 if v in ("vae", "ae") else 0.0) for v in variants}
    hp_d = dict(hps, **({"w": gm_b200.AdamHP.make(LR["w"], clamp=0.01)} if "w" in variants else {}))

    def step(name, s):
        eng, hp = engines[name], hps[name]
        x = pool[(s % 4) * B * 4096:(s % 4 + 1) * B * 4096]
        if name == "vae":
            eng.vae_grad(x, B, seed=1000, step=s)              # compute_batch + (recon + kl).backward(), optimizer.step()
            eng.apply(hp)
            return
        if name == "ae":
            eng.ae_grad(x, B)                                   # compute_batch + recon.backward(), optimizer.step()
            eng.apply(hp)
            return
        eng.d_grad(x, B, seed=1000, step=s)
        eng.apply(1, hp_d[name])
        eng.g_grad(B, seed=1000, step=s)
        eng.apply(0, hp)
        if name == "be":
            eng.began_control(0.5, 1e-3, 5 * 4)                 # GAMMA, LAMBDA, patience 5 len(train_iter) of src/be_gan.py
        if name == "info":
            eng.q_grad(B, seed=1000, step=s)                    # the MI step and MI_optimizer (src/info_gan.py:196-205)
            eng.apply_mi(hp)

    launches = {}
    for name in variants:
        step(name, 0)
        torch.cuda.synchronize()
        gm_b200.launch_count(reset=True)
        step(name, 1)
        torch.cuda.synchronize()
        launches[name] = gm_b200.launch_count(reset=True)
    for s in range(a.warmup):
        for name in variants:
            step(name, 2 + s)
    torch.cuda.synchronize()
    ms = {name: [] for name in variants}
    for s in range(a.steps):
        for name in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(name, 100 + s)
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    out = {}
    for name in variants:
        med = sorted(ms[name])[len(ms[name]) // 2]
        if name == "be":
            flop = began_flop_per_img()
        elif name == "info":
            flop = info_flop_per_img()
        elif name == "vae":
            flop = vae_flop_per_img()
        elif name == "ae":
            flop = vae_flop_per_img(z=AE_Z, heads=1)
        else:
            flop = _dcgan_flop_per_img() + (4 * critic_flop_per_img() if name in ("wgp", "dra") else 0.0)
        out[name] = {"median_ms": round(med, 3), "min_ms": round(min(ms[name]), 3), "images_per_s": round(B / med * 1e3, 1),
                     "launches_per_step": launches[name], "gflop_per_image": round(flop / 1e9, 3),
                     "tflops": round(flop * B / med / 1e9, 1),
                     "last_losses": [float(v) for v in {"vae": engines[name].vae_loss, "ae": engines[name].ae_loss}.get(
                         name, engines[name].loss_buf).tolist()]}
    for name in variants[1:]:
        out[name]["over_ns_images_per_s"] = round(out[name]["images_per_s"] / out["ns"]["images_per_s"], 3)
    if variants is not GROUPS[0]:                               # the first group's NSGAN leg keeps the "ns" key
        out["ns_group2"] = out.pop("ns")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    dev = torch.cuda.current_device()
    B = a.batch
    g = torch.Generator(device="cuda").manual_seed(77)
    pool = (torch.rand(4 * B * 4096, 3, device="cuda", generator=g) < 0.3).to(torch.bfloat16)
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit(dev), "batch": B, "steps": a.steps,
           "warmup": a.warmup}
    for group in GROUPS:
        out.update(run_group(group, a, pool))
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
