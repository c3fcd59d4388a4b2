"""The 128 x 208 MN-major GEMM route (GPU): split-K weight gradients whose covered columns need an even number of 208-wide
n-tiles and no more than 256-wide ones (N = 400 and 401 in the train steps) take the 208-wide tile, as 2-CTA clusters
over n-tile pairs; every other wide TN product keeps the 256-wide tile.  Each case is judged per element against float64 with
the bounds of test_gemm_conformance_gpu, the tile width it must take is read from the level-2 profile, and the route
must reproduce the 256-wide one (GM_TN208=0) bit for bit: the tile and split counts are the same, so every output
element sums the same k-blocks in the same order.  That holds for the bare GEMMs and for the parameters, Adam moments
and losses after two seeded steps of NSGAN, WGAN-GP and the VAE."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gemm_conformance_gpu as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X, H, Z = 784, 400, 20

# (M, N, K, transpose, ldc, tile width).  The step's dW1d over 2B and 3B rows (B = 65536; WGAN-GP appends the penalty's
# rows) and dW2g over B rows, the VAE's 131072-row weight gradients, ragged K, odd 208-wide n-tile counts (N = 100, 208
# and 624 keep the 256-wide tile), N = 209 and 256 (one 256-wide tile is fewer than two 208-wide ones), 81 m-tiles over
# the clusters the device holds at once, and N = 832 (two n-tile pairs).
SHAPES = [(785, 400, 2 * 65536, True, 800, 208), (785, 400, 3 * 65536, True, 800, 208), (784, 401, 65536, False, 448, 208),
          (784, 401, 131072, False, 404, 208), (785, 400, 4129, True, 785, 208), (100, 401, 1000, False, 401, 208),
          (300, 100, 3000, False, 100, 256), (129, 208, 777, True, 136, 256), (785, 624, 1024, False, 624, 256),
          (200, 209, 2000, False, 216, 256), (130, 256, 1500, True, 130, 256), (128 * 80 + 5, 400, 256, False, 400, 208),
          (785, 832, 2048, False, 832, 208)]
CASES = [dict(C._f32_case(50 + i, "tn", M, N, K, tr, ldc, True), width=w) for i, (M, N, K, tr, ldc, w) in enumerate(SHAPES)]


def _widths(c):
    """-> (tensors, tile widths of the TN GEMM launches) of one run under the level-2 profile"""
    import gm_b200
    T = C._tensors(c)
    torch.cuda.synchronize()
    gm_b200.prof_report()
    gm_b200.prof_enable(2)
    try:
        C._launch(c, T)
        names = [n for n, _, _ in gm_b200.prof_report() if n.startswith("gemm_tn")]
    finally:
        gm_b200.prof_enable(0)
    return T, [int(n[len("gemm_tn"):n.index("[")]) for n in names]


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_tn_gemm_matches_float64(c):
    T, counts, _ = C._run_counted(c)
    assert counts == [0, 0, 1, 0], (c["name"], counts)       # both widths count as the wide TN kind
    C._check(c, T)
    del T
    T, widths = _widths(c)
    assert widths == [c["width"]], (c["name"], widths)


def test_repeated_calls_give_identical_bits():
    for c in CASES[:3] + CASES[8:9] + CASES[11:]:
        T1, T2 = C._run(c), C._run(c)
        assert torch.equal(T1["out"].view(torch.int32), T2["out"].view(torch.int32)), c["name"]


def _pool(n, seed=3435):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n, X // 8), device="cuda", dtype=torch.uint8, generator=g)


def _train_states():
    """parameters, Adam moments and losses after two seeded steps of NSGAN, WGAN-GP (B = 65536) and the VAE (131072)"""
    import gm_b200
    import torch.nn as nn
    hp = gm_b200.AdamHP.make(2e-4)
    res = {}
    for variant in ("ns", "wgp"):
        B, N, seed = 65536, 2 * 65536, 99
        eng = gm_b200.GanEngine(X, H, Z, max_batch=B, variant=variant, d_out_act="relu" if variant == "wgp" else "sigmoid")
        torch.manual_seed(1234)
        g1, g2, d1, d2 = nn.Linear(Z, H), nn.Linear(H, X), nn.Linear(X, H), nn.Linear(H, 1)
        eng.load(0, [g1.weight.data, g1.bias.data, g2.weight.data, g2.bias.data])
        eng.load(1, [d1.weight.data, d1.bias.data, d2.weight.data, d2.bias.data])
        eng.set_sampler(N, seed)
        bits = _pool(N)
        losses = []
        for s in range(2):
            losses.append(eng.d_grad(bits, fmt="bits", batch=B, seed=seed, step=s).clone())
            eng.apply(1, hp)
            losses.append(eng.g_grad(B, seed=seed, step=s).clone())
            eng.apply(0, hp)
        torch.cuda.synchronize()
        for net in (0, 1):
            for k, t in (("params", eng.params), ("m", eng.exp_avg), ("v", eng.exp_avg_sq)):
                res["%s_%s%d" % (variant, k, net)] = t[net].view(torch.int32).cpu().numpy()
        res[variant + "_losses"] = torch.cat([l.reshape(-1) for l in losses]).view(torch.int32).cpu().numpy()
        del eng
    B, N, seed = 131072, 2 * 131072, 77
    eng = gm_b200.VaeEngine(X, H, Z, max_batch=B)
    torch.manual_seed(1234)
    mods = {"encoder.linear": nn.Linear(X, H), "encoder.mu": nn.Linear(H, Z), "encoder.log_var": nn.Linear(H, Z),
            "decoder.linear": nn.Linear(Z, H), "decoder.recon": nn.Linear(H, X)}
    t = {}
    for k, m in mods.items():
        t[k + ".weight"], t[k + ".bias"] = m.weight.data, m.bias.data
    eng.load(t)
    eng.set_sampler(N, N // B, seed)
    bits = _pool(N)
    losses = []
    for s in range(2):
        losses.append(eng.grad(bits, fmt="bits", batch=B, seed=seed, step=s).clone())
        eng.apply(hp)
    torch.cuda.synchronize()
    for k, v in (("params", eng.params), ("m", eng.exp_avg), ("v", eng.exp_avg_sq)):
        res["vae_" + k] = v.view(torch.int32).cpu().numpy()
    res["vae_losses"] = torch.cat(losses).view(torch.int32).cpu().numpy()
    return res


def _outputs():
    res = {}
    for c in CASES:
        res[c["name"]] = C._run(c)["out"].view(torch.int32).cpu().numpy()
    res.update(_train_states())
    return res


def _dump(path):
    np.savez(path, **_outputs())


def test_outputs_match_the_256_wide_route_bit_for_bit(tmp_path):
    """every case above and the three train steps again in a fresh process with GM_TN208=0: the same bits"""
    path = str(tmp_path / "out.npz")
    env = dict(os.environ, GM_TN208="0")
    paths = [ROOT, os.path.join(ROOT, "generative-models_b200"), os.path.join(ROOT, "tests")]
    env["PYTHONPATH"] = os.pathsep.join(paths + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    code = "import test_gemm_tn208_gpu as T; T._dump(%r)" % path
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    other = np.load(path)
    mine = _outputs()
    assert sorted(other.files) == sorted(mine)
    diff = [k for k in mine if not np.array_equal(mine[k], other[k])]
    assert not diff, diff
