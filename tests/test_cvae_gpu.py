"""Conditional VAE on the GPU: the fused CVAE step (gm_cvae_grad) against the float64 oracle (tests/cvae_oracle.py) at its
bf16 points, a CVAE with zero label weights against the VAE engine bit for bit, the resident (image, label) draw, the
forward-only entries, the per-call encoder / decoder under a user-written compute_batch, CVAETrainer.train, and the C
ABI's refusals and launch ledger.

Bounds are test_vae_gpu.py's and test_bir_vae_gpu.py's: losses within 1e-3 relative; gradients within 3e-3 norm-relative
of the oracle evaluated at the engine's own bf16 storage points (the remaining error is the fp32 accumulation order of
the GEMMs and split-K partials); forward outputs within test_vae_gpu.py's 5e-3 of an fp32 torch evaluation."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gm_b200
from gm_b200 import GmError
from cvae_oracle import cvae_step
from mlp_harness import VaeReluSides, nrel
from inputs import gm_init_weights
from oracle import ref_math as R

pytestmark = pytest.mark.gpu


def _weights(X, H, Z, K, seed):
    shapes = [("encoder.linear", (H, X + K)), ("encoder.mu", (Z, H)), ("encoder.log_var", (Z, H)),
              ("decoder.linear", (H, Z + K)), ("decoder.recon", (X, H))]
    W = gm_init_weights(shapes, seed)
    return {k + s: v for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))}


def _labels(rng, b, K):
    y = rng.integers(0, K, b)
    y[:min(b, K)] = np.arange(min(b, K))
    return y


GEOMS = [(784, 400, 20, 10), (208, 208, 7, 5), (784, 400, 20, 43)]


@pytest.mark.parametrize("geom", GEOMS, ids=["%dx%dx%dc%d" % g for g in GEOMS])
def test_fused_step_against_the_oracle(geom):
    X, H, Z, K = geom
    eng = gm_b200.CvaeEngine(X, H, Z, K, max_batch=4096)
    eng.load(_weights(X, H, Z, K, 91 + Z + K))
    rng = np.random.default_rng(X + H + Z + K)
    P = {k: v.double().cpu().numpy() for k, v in eng.views().items()}
    for b in (1, 65, 300, 4096):
        x = (rng.random((b, X)) < 0.13).astype(np.float32)
        y = _labels(rng, b, K)
        eps = rng.standard_normal((b, Z)).astype(np.float32)
        ls = eng.grad(torch.from_numpy(x).cuda(), torch.from_numpy(y), eps=torch.from_numpy(eps).cuda()).cpu().numpy()
        sides = VaeReluSides(eng)
        recon, kl, g, _ = cvae_step(P, x.astype(np.float64), y, eps.astype(np.float64), K, q=R.bf16_points, relu=sides)
        assert abs(ls[0] - recon) <= 1e-3 * recon, (b, ls[0], recon)
        assert abs(ls[1] - kl) <= 1e-3 * kl, (b, ls[1], kl)
        # the staged rows carry the one-hot and the ones column
        xin = eng.debug_read("Xin", 0, b, X + K + 1).cpu().numpy()
        assert np.array_equal(xin[:, X:X + K], np.eye(K)[y]) and (xin[:, X + K] == 1).all()
        zb = eng.debug_read("Zb", 0, b, 64).cpu().numpy()
        assert np.array_equal(zb[:, Z:Z + K], np.eye(K)[y]) and (zb[:, Z + K] == 1).all() and not zb[:, Z + K + 1:].any()
        gv = {k: v.cpu().numpy() for k, v in eng.views(eng.grads).items()}
        for k in g:
            assert nrel(gv[k], g[k]) < 3e-3, (b, k, nrel(gv[k], g[k]))


def test_zero_label_weights_are_the_vae_bit_for_bit():
    """Every GEMM keeps the VAE's tile grid, k-block count and split-K split: e1 contracts over 800 columns instead of
    784, but both are 13 k-blocks of 64 and the extra products are exact zeros (zero weights), so each fp32 sum is the
    same.  Hence the losses and every shared gradient are bitwise the VAE's, with fixed or in-kernel eps."""
    X, H, Z, K = 784, 400, 20, 10
    vae_w = _weights(X, H, Z, 0, 5)
    cw = dict(vae_w)
    for k in ("encoder.linear.weight", "decoder.linear.weight"):
        cw[k] = np.concatenate([vae_w[k], np.zeros((H, K), np.float32)], axis=1)
    ve, ce = gm_b200.VaeEngine(X, H, Z, max_batch=512), gm_b200.CvaeEngine(X, H, Z, K, max_batch=512)
    ve.load(vae_w)
    ce.load(cw)
    rng = np.random.default_rng(1)
    for b in (1, 65, 512):
        x = torch.from_numpy((rng.random((b, X)) < 0.13).astype(np.float32)).cuda()
        y = torch.from_numpy(_labels(rng, b, K))
        eps = torch.from_numpy(rng.standard_normal((b, Z)).astype(np.float32)).cuda()
        for e in (eps, None):
            lv = ve.grad(x, eps=e, seed=3, step=b).clone()
            lc = ce.grad(x, y, eps=e, seed=3, step=b).clone()
            assert torch.equal(lv, lc), (b, lv, lc)
            gv, gc = ve.views(ve.grads), ce.views(ce.grads)
            for k in gv:
                a = gc[k][:, :gv[k].shape[1]] if k in ("encoder.linear.weight", "decoder.linear.weight") else gc[k]
                assert torch.equal(a, gv[k]), (b, k)
            assert torch.equal(ve.last_eps(b), ce.last_eps(b))


def test_resident_draws_the_host_gathers_pairs():
    X, H, Z, K, n, bs = 784, 400, 20, 10, 1000, 300
    eng = gm_b200.CvaeEngine(X, H, Z, K, max_batch=bs)
    eng.load(_weights(X, H, Z, K, 3))
    g = torch.Generator().manual_seed(2)
    imgs = (torch.rand(n, X, generator=g) < 0.13).float()
    labels = torch.randint(0, K, (n,), generator=g)
    bits = gm_b200.gan_api.DeviceDataset(imgs, bs).bits
    bpe, seed = -(-n // bs), 77
    yd = eng.class_ids(labels)
    for step in (0, 3, 5):
        rows = min(bs, n - (step % bpe) * bs)
        eng.set_sampler(n, bpe, seed, batch_size=bs)
        l1 = eng.grad(bits, yd, fmt="bits", batch=rows, seed=9, step=step).clone()
        g1, eps, xin1 = eng.grads.clone(), eng.last_eps(rows), eng.debug_read("Xin", 0, rows, X + K + 1)
        eng.set_sampler(0, 0, 0)
        idx = eng.sample_indices(bs, step, bpe, n, seed)[:rows]           # batch k starts at row k * bs of the permutation
        assert len(set(idx.tolist())) == rows
        l2 = eng.grad(imgs.cuda(), labels, eps=eps, gather_idx=idx).clone()
        assert torch.equal(l1, l2) and torch.equal(g1, eng.grads)
        assert torch.equal(xin1, eng.debug_read("Xin", 0, rows, X + K + 1))
        assert torch.equal(xin1[:, X:X + K].argmax(1).cpu(), labels[idx.long().cpu()])


def test_forward_decode_and_evaluate_against_the_oracle():
    import cvae
    X, H, Z, K, b = 784, 400, 20, 10, 512
    eng = gm_b200.CvaeEngine(X, H, Z, K, max_batch=b)
    eng.load(_weights(X, H, Z, K, 11))
    rng = np.random.default_rng(4)
    x = (rng.random((b, X)) < 0.13).astype(np.float32)
    y = _labels(rng, b, K)
    eps = rng.standard_normal((b, Z)).astype(np.float32)
    out, mu, lv, ls = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(y), eps=torch.from_numpy(eps).cuda(),
                                  want_losses=True)
    P = {k: v.double().cpu().numpy() for k, v in eng.views().items()}
    recon, kl, _, fw = cvae_step(P, x.astype(np.float64), y, eps.astype(np.float64), K)
    assert nrel(mu.cpu().numpy(), fw["mu"]) < 5e-3 and nrel(lv.cpu().numpy(), fw["lv"]) < 5e-3
    assert nrel(out.cpu().numpy(), fw["out"]) < 5e-3
    assert abs(ls[0].item() - recon) <= 2e-3 * recon and abs(ls[1].item() - kl) <= 2e-3 * kl
    z = torch.from_numpy(fw["z"].astype(np.float32)).cuda()
    d1 = eng.decode(z, torch.from_numpy(y))
    d2 = eng.decode(z, torch.from_numpy(y))
    assert torch.equal(d1, d2)                                             # the same (z, y) decodes to the same bits
    assert nrel(d1.cpu().numpy(), fw["out"]) < 5e-3
    # the label changes the decoded image
    assert not torch.equal(d1, eng.decode(z, torch.from_numpy((y + 1) % K)))
    # evaluate: the mean per-batch loss of the forward-only path
    model = cvae.CVAE(X, H, Z, K)
    sd = {k: torch.from_numpy(v.astype(np.float32)) for k, v in _weights(X, H, Z, K, 11).items()}
    model.load_state_dict(sd)
    loader = [(torch.from_numpy(x).view(b, 1, 28, 28), torch.from_numpy(y))]
    tr = cvae.CVAETrainer(model, loader, loader, loader)
    torch.manual_seed(8)
    val = tr.evaluate(loader)
    torch.manual_seed(8)
    e8 = torch.randn(b, Z).double().numpy()
    r8, k8, _, _ = cvae_step(P, x.astype(np.float64), y, e8, K)
    assert abs(val - (r8 + k8)) <= 2e-3 * (r8 + k8)


def _q(t):
    """t rounded to bf16 in the forward, the identity in the backward"""
    return t + (t.to(torch.bfloat16).double() - t).detach()


def _torch64(P, x, y, eps, K):
    """the CVAE forward in float64 torch autograd at the device's bf16 storage points (test_vae_custom_gpu.py's): the
    weights, x, the hidden rows, z and the returned images.  The images matter for a BCE: its upstream
    (out - x) / (out (1 - out)) is taken at the bf16 image the decoder returns."""
    W = {k: _q(v) if k.endswith("weight") else v for k, v in P.items()}
    Y = F.one_hot(y, K).double()
    h1 = _q(torch.relu(torch.cat([_q(x), Y], 1) @ W["encoder.linear.weight"].t() + W["encoder.linear.bias"]))
    mu = h1 @ W["encoder.mu.weight"].t() + W["encoder.mu.bias"]
    lv = h1 @ W["encoder.log_var.weight"].t() + W["encoder.log_var.bias"]
    z = _q(mu + eps * torch.exp(lv / 2))
    h3 = _q(torch.relu(torch.cat([z, Y], 1) @ W["decoder.linear.weight"].t() + W["decoder.linear.bias"]))
    return _q(torch.sigmoid(h3 @ W["decoder.recon.weight"].t() + W["decoder.recon.bias"])), mu, lv


def _bce_beta4():
    def compute_batch(self, batch):
        images, labels = batch
        images = images.view(images.shape[0], -1).cuda()
        out, mu, log_var = self.model(images, labels)
        recon = F.binary_cross_entropy(out, images, reduction="sum")
        return recon, 4.0 * self.kl_divergence(mu, log_var)
    return compute_batch


def test_custom_compute_batch_bce_beta4_matches_float64_autograd(capsys):
    import cvae
    X, H, Z, K, b = 784, 400, 20, 10, 65
    torch.manual_seed(6)
    model = cvae.CVAE(X, H, Z, K)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.uniform_(-0.1, 0.1)
    x = (torch.rand(b, 1, 28, 28) < 0.3).float()
    y = torch.randint(0, K, (b,))
    loader = [(x, y)]
    Custom = type("Custom", (cvae.CVAETrainer,), {"compute_batch": _bce_beta4()})
    tr = Custom(model, loader, loader, loader)
    P = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(12)
    recon, kl = tr.compute_batch(loader[0])
    (recon + kl).backward()
    torch.manual_seed(12)
    eps = torch.randn(b, Z).double()
    out, mu, lv = _torch64(P, x.view(b, -1).double(), y, eps, K)
    recon64 = F.binary_cross_entropy(out, x.view(b, -1).double(), reduction="sum")
    kl64 = 4.0 * torch.sum(0.5 * (mu ** 2 + torch.exp(lv) - lv - 1))
    (recon64 + kl64).backward()
    assert abs(recon.item() - recon64.item()) <= 1e-2 * recon64.item() and abs(kl.item() - kl64.item()) <= 1e-2 * kl64.item()
    # test_vae_custom_gpu.py's bound for the MLP VAE's per-call backward against this restatement
    for k, p in model.named_parameters():
        assert nrel(p.grad.double().cpu().numpy(), P[k].grad.numpy()) < 2e-2, (k, nrel(p.grad.double().cpu().numpy(), P[k].grad.numpy()))
    # and train() runs the reference loop over the override
    tr.train(num_epochs=2, lr=1e-3, weight_decay=1e-5)
    assert "Epoch[2/2], Total Loss: " in capsys.readouterr().out
    assert len(tr.recon_loss) == len(tr.kl_loss) == 2 and tr.recon_loss[1] < tr.recon_loss[0]


def test_overwritten_slots_and_double_backward_raise():
    import cvae
    model = cvae.CVAE(784, 64, 8, 4)
    loader = [(torch.zeros(4, 1, 28, 28), torch.zeros(4, dtype=torch.long))]
    tr = cvae.CVAETrainer(model, loader, loader, loader)
    tr._ensure_engine(4)
    x, y = torch.rand(4, 784).cuda(), torch.tensor([0, 1, 2, 3])
    mu0, _ = model.encoder(x, y)
    model.encoder(x, y)
    model.encoder(x, y)                                           # two slots: the first call's activations are gone
    with pytest.raises(RuntimeError, match="overwritten"):
        mu0.sum().backward()
    z = torch.randn(4, 8, device="cuda", requires_grad=True)
    out = model.decoder(z, y)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(out.sum(), list(model.decoder.parameters()), create_graph=True)
    with pytest.raises(GmError, match=r"in \[0, 4\)"):
        model.decoder(z, torch.tensor([0, 1, 2, 4]))


def test_trainer_trains_one_epoch_on_get_data(capsys):
    import cvae
    from utils import get_data
    train_iter, val_iter, test_iter = get_data()
    model = cvae.CVAE(784, 400, 20, 10)
    tr = cvae.CVAETrainer(model, train_iter, val_iter, test_iter)
    tr.train(1)
    out = capsys.readouterr().out
    assert "Epoch[1/1], Total Loss: " in out and ", Reconst Loss: " in out and ", KL Div: " in out and ", Val Loss: " in out
    nb = len(train_iter)
    assert tr._resident is not None and len(tr.recon_loss) == len(tr.kl_loss) == nb
    assert all(np.isfinite(tr.recon_loss + tr.kl_loss))
    assert np.mean(tr.recon_loss[-50:]) < np.mean(tr.recon_loss[:50])
    assert isinstance(tr.best_model, cvae.CVAE) and tr.best_model is not model
    s = tr.sample_images(num_images=36)
    assert s.shape == (36, 28, 28) and torch.isfinite(s).all()
    for c in range(10):
        sc = tr.sample_images(num_images=5, labels=torch.full((5,), c))
        assert sc.shape == (5, 28, 28)
    imgs, labels = next(iter(test_iter))
    assert tr.reconstruct_images(imgs[:8], labels[:8], 0).shape == (8, 28, 28)


def _rc(fn, *a):
    from gm_b200._lib import lib
    return getattr(lib(), fn)(*a)


def test_c_abi_refuses_bad_arguments_before_any_launch():
    from gm_b200._lib import ctx, VaeDesc
    h = ctx()
    vp = C.c_void_p
    out = C.c_void_p()
    for d, k in [(VaeDesc(784, 400, 20, 8, 0), 0), (VaeDesc(784, 400, 20, 8, 0), 44), (VaeDesc(784, 400, 33, 8, 0), 10),
                 (VaeDesc(784, 448, 20, 8, 0), 10), (VaeDesc(784, 400, 20, 8, 1), 10), (VaeDesc(780, 400, 20, 8, 0), 10)]:
        assert _rc("gm_cvae_create", h, C.byref(d), k, C.byref(out)) != 0, (d.z_dim, k)
    eng = gm_b200.CvaeEngine(784, 400, 20, 10, max_batch=8)
    vae = gm_b200.VaeEngine(784, 400, 20, max_batch=8)
    x = torch.zeros(8, 784, device="cuda")
    y = torch.zeros(8, dtype=torch.int32, device="cuda")
    ml = torch.zeros(8, 40, device="cuda")
    px, py, pm = vp(x.data_ptr()), vp(y.data_ptr()), vp(ml.data_ptr())
    n0 = gm_b200.launch_count()
    g = eng.g
    bad = [("gm_cvae_grad", (g, px, 0, None, None, 8, None, 0, 0, None, None)),
           ("gm_cvae_grad", (g, None, 0, py, None, 8, None, 0, 0, None, None)),
           ("gm_cvae_grad", (g, px, 1, py, None, 8, None, 0, 0, None, None)),
           ("gm_cvae_grad", (g, px, 0, py, None, 9, None, 0, 0, None, None)),
           ("gm_cvae_grad", (g, px, 0, py, None, 0, None, 0, 0, None, None)),
           ("gm_cvae_grad", (g, px, 0, vp(y.data_ptr() + 2), None, 8, None, 0, 0, None, None)),
           ("gm_cvae_grad", (vae.g, px, 0, py, None, 8, None, 0, 0, None, None)),
           ("gm_cvae_forward", (g, px, 0, None, 8, None, 0, 0, None, pm, None, None)),
           ("gm_cvae_forward", (vae.g, px, 0, py, 8, None, 0, 0, None, pm, None, None)),
           ("gm_cvae_decode", (g, px, py, 8, None, None)),
           ("gm_cvae_decode", (g, px, None, 8, px, None)),
           ("gm_cvae_encoder_forward", (g, 2, px, py, 8, pm, None)),
           ("gm_cvae_encoder_forward", (g, 0, px, py, 9, pm, None)),
           ("gm_cvae_encoder_forward", (g, 0, px, None, 8, pm, None)),
           ("gm_cvae_decoder_forward", (g, -1, px, py, 8, px, None)),
           ("gm_cvae_decoder_forward", (vae.g, 0, px, py, 8, px, None)),
           ("gm_vae_grad", (g, px, 0, None, 8, None, 1.0, 0, 0, None, None)),
           ("gm_vae_forward", (g, px, 0, 8, None, 0, 0, None, pm, None, None)),
           ("gm_vae_decode", (g, px, 8, px, None)),
           ("gm_vae_encoder_forward", (g, 0, px, 8, pm, None)),
           ("gm_vae_decoder_forward", (g, 0, px, 8, px, None))]
    for fn, a in bad:
        assert _rc(fn, *a) != 0, fn
    assert gm_b200.launch_count() == n0
    with pytest.raises(GmError, match="integer"):
        eng.grad(x, torch.zeros(8))
    with pytest.raises(GmError, match="labels for 8 rows"):
        eng.grad(x, torch.zeros(7, dtype=torch.long))
    assert gm_b200.launch_count() == n0


def test_wrong_shaped_labels_are_refused_before_any_launch():
    """one-hot matrices and label vectors of the wrong length, at every entry that takes labels: the model's calls, the
    trainer's host and resident paths, sampling, and the engine's gathered and sampled steps"""
    import cvae
    K, n = 10, 8
    model = cvae.CVAE(784, 64, 8, K)
    x = (torch.rand(n, 1, 28, 28) < 0.13).float()
    y = torch.arange(n) % K
    tr = cvae.CVAETrainer(model, [(x, y)], [(x, y)], [(x, y)])
    eng = tr._ensure_engine(n)
    onehot = F.one_hot(y, K)
    for call in (lambda: model(x.view(n, -1), onehot), lambda: model.encoder(x.view(n, -1), onehot),
                 lambda: model.decoder(torch.randn(n, 8), onehot), lambda: tr.compute_batch((x, onehot)),
                 lambda: tr.evaluate([(x, onehot)])):
        with pytest.raises(GmError, match="shape"):
            call()
    for call in (lambda: model(x.view(n, -1), torch.arange(n + 1) % K), lambda: tr.compute_batch((x, y[:n - 1])),
                 lambda: tr.sample_images(num_images=4, labels=torch.arange(5) % K)):
        with pytest.raises(GmError, match="labels for"):
            call()
    with torch.no_grad():
        with pytest.raises(GmError, match="shape"):
            model(x.view(n, -1), onehot)
    pool = (torch.rand(100, 784, device="cuda") < 0.13).float()
    idx = torch.arange(n, dtype=torch.int32, device="cuda")
    n0 = gm_b200.launch_count()
    with pytest.raises(GmError, match="99 labels for 100 rows"):        # gather_idx: one label per pool image
        eng.grad(pool, torch.arange(99) % K, gather_idx=idx)
    eng.set_sampler(100, 12, 1, batch_size=n)
    try:
        with pytest.raises(GmError, match="8 labels for 100 rows"):     # the sampler: one label per pool image
            eng.grad(pool, y, batch=n)
    finally:
        eng.set_sampler(0, 0, 0)
    assert gm_b200.launch_count() == n0
    imgs = (torch.rand(64, 1, 28, 28) < 0.13).float()
    bad = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, F.one_hot(torch.arange(64) % K, K)), batch_size=32)
    tr2 = cvae.CVAETrainer(cvae.CVAE(784, 64, 8, K), bad, bad, bad)
    with pytest.raises(GmError, match="shape"):                          # the resident path's label upload
        tr2.train(1)
    assert tr2._engine is None


def test_launch_ledger_of_the_new_entries():
    eng = gm_b200.CvaeEngine(784, 400, 20, 10, max_batch=64)
    x = (torch.rand(64, 784, device="cuda") < 0.13).float()
    y = torch.arange(64) % 10
    gm_b200.prof_enable(2)
    try:
        eng.grad(x, y)
        eng.forward(x, y, want_losses=True)
        eng.decode(torch.randn(64, 20, device="cuda"), y)
        eng.encoder_forward(0, x, y)
        eng.decoder_forward(0, torch.randn(64, 20, device="cuda"), y)
        torch.cuda.synchronize()
        names = {n: c for n, c, _ in gm_b200.prof_report()}
    finally:
        gm_b200.prof_enable(0)
    assert names.get("cvae_stage_kernel", 0) == 3, names
    assert names.get("cvae_reparam_kernel", 0) == 2, names
    assert names.get("cvae_latent_rows_kernel", 0) == 2, names
    for k in ("stage_images_kernel", "vae_reparam_kernel", "stage_noise_kernel"):
        assert names.get(k, 0) == 0, (k, names)
