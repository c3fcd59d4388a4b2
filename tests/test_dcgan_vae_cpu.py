"""The VAE on the DCGAN conv path, CPU side: the decomposition the device runs (closed-form dpre through the sigmoid, the
decoder backward to dz, the (dmu, dlv) formula, the encoder backward; tests/dcgan_vae_oracle.py) against float64 autograd of
src/vae.py's compute_batch on the conv VAE, and the surface of the dc_vae drop-in.  No GPU needed."""
import inspect

import pytest
import torch

import dcgan_vae_oracle as VO


def _nets(hd=8, z=6, seed=0, wstd=0.05):
    torch.manual_seed(seed)
    E, G = VO.Encoder(hd, z).double(), VO.Decoder(hd, z).double()
    with torch.no_grad():
        for net in (E, G):
            for name, p in net.named_parameters():
                if name.split(".")[-2].startswith("l"):
                    p.normal_(0.0, wstd)
    E.train(); G.train()
    return E, G


@pytest.mark.parametrize("seed,binary", [(0, True), (1, False)])
def test_vae_step_decomposition_equals_float64_autograd(seed, binary):
    z, n = 6, 5
    E, G = _nets(z=z, seed=seed)
    g = torch.Generator().manual_seed(seed + 3)
    x = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    if binary:
        x = (x < 0.3).double()
    eps = torch.randn(n, z, generator=g, dtype=torch.float64)
    pE, pG = list(E.parameters()), list(G.parameters())
    recon, kl = VO.compute_batch(E, G, x, eps)
    ref = torch.autograd.grad(recon + kl, pE + pG)
    recon, kl = recon.detach(), kl.detach()
    # the device's order: encoder heads, z, decoder to the pre-sigmoid output, closed-form dpre, decoder backward to dz,
    # (dmu, dlv), encoder backward
    heads = E.heads(x)
    mu, lv = heads[:, :z].detach(), heads[:, z:].detach()
    zz = VO.reparameterize(mu, lv, eps).requires_grad_(True)
    pre = G.pre(zz)
    out = torch.sigmoid(pre).detach().reshape(n, -1)
    got_recon = float(((x - out) ** 2).sum())
    got_kl = float(VO.kl_divergence(mu, lv))
    assert abs(got_recon - float(recon)) <= 1e-12 * abs(float(recon)) and abs(got_kl - float(kl)) <= 1e-12 * abs(float(kl))
    dp = VO.dpre(out, x).view(pre.shape)
    *gG, dz = torch.autograd.grad(pre, pG + [zz], dp)
    dmu, dlv = VO.dlatent(mu, lv, eps, dz)
    gE = torch.autograd.grad(heads, pE, torch.cat([dmu, dlv], 1))
    names = ["encoder." + k for k, _ in E.named_parameters()] + ["decoder." + k for k, _ in G.named_parameters()]
    assert len(names) == 11 + 13
    for name, a, b in zip(names, list(gE) + list(gG), ref):
        rel = float((a - b).norm() / b.norm().clamp_min(1e-300))
        assert rel <= 1e-9, (name, rel)


def _sig(fn):
    return [(k, v.default) for k, v in inspect.signature(fn).parameters.items()][1:]


def test_dc_vae_surface_without_a_gpu():
    import dc_vae as M
    from gm_b200 import GmError
    E = inspect.Parameter.empty
    # src/vae.py:84,110,127,193,210,214,225,254,278,295,336,348,367,371
    assert _sig(M.DCVAE.__init__) == [("image_size", 64 * 64 * 3), ("hidden_dim", 64), ("z_dim", 100), ("channels", 3)]
    assert _sig(M.DCVAETrainer.__init__) == [("model", E), ("train_iter", E), ("val_iter", E), ("test_iter", E), ("viz", False)]
    assert _sig(M.DCVAETrainer.train) == [("num_epochs", E), ("lr", 1e-3), ("weight_decay", 1e-5)]
    assert _sig(M.DCVAETrainer.compute_batch) == [("batch", E)]
    assert _sig(M.DCVAETrainer.kl_divergence) == [("mu", E), ("log_var", E)]
    assert _sig(M.DCVAETrainer.evaluate) == [("iterator", E)]
    assert _sig(M.DCVAETrainer.reconstruct_images) == [("images", E), ("epoch", E), ("save", True)]
    assert _sig(M.DCVAETrainer.sample_images) == [("epoch", -100), ("num_images", 36), ("save", True)]
    assert _sig(M.DCVAETrainer.explore_latent_space) == [("num_epochs", 3)]
    for fn in ("sample_interpolated_images", "make_all", "viz_loss", "save_model", "load_model"):
        assert callable(getattr(M.DCVAETrainer, fn))
    model = M.DCVAE(image_size=64 * 64 * 3, hidden_dim=16, z_dim=20)
    assert (model.image_size, model.hidden_dim, model.z_dim, model.shape) == (12288, 16, 20, 64)
    sd = model.state_dict()
    bn = lambda pfx, i: ["%s.bn%d.%s" % (pfx, i, k) for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]  # noqa: E731
    enc = (["encoder.l%d.weight" % i for i in range(1, 5)] + sum((bn("encoder", i) for i in (2, 3, 4)), [])
           + ["encoder.mu.weight", "encoder.log_var.weight"])
    dec = ["decoder.l%d.weight" % i for i in range(1, 6)] + sum((bn("decoder", i) for i in (1, 2, 3, 4)), [])
    assert list(sd) == enc + dec
    shapes = {"encoder.l1.weight": (16, 3, 4, 4), "encoder.l4.weight": (128, 64, 4, 4), "encoder.mu.weight": (20, 128, 4, 4),
              "encoder.log_var.weight": (20, 128, 4, 4), "encoder.bn2.weight": (32,), "decoder.l1.weight": (20, 128, 4, 4),
              "decoder.l2.weight": (128, 64, 4, 4), "decoder.l5.weight": (16, 3, 4, 4), "decoder.bn4.running_var": (16,)}
    for k, shp in shapes.items():
        assert tuple(sd[k].shape) == shp, k
    assert not any(k.endswith(".bias") and ".bn" not in k for k in sd)                   # every conv is bias-free
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCVAETrainer(model, it, it, it)
    assert tr.name == "DCVAE" and tr.kl_loss == [] and tr.recon_loss == [] and tr.best_val_loss == 1e10
    mu, lv = torch.randn(4, 20, dtype=torch.float64), torch.randn(4, 20, dtype=torch.float64)
    assert float(tr.kl_divergence(mu, lv)) == pytest.approx(float(VO.kl_divergence(mu, lv)))
    with pytest.raises(GmError):
        M.DCVAE(image_size=784)
    with pytest.raises(GmError):
        M.DCVAE(hidden_dim=24)
    with pytest.raises(GmError):
        tr.explore_latent_space()
    with pytest.raises(GmError):
        tr.make_all()
    if not torch.cuda.is_available():   # no GPU: a loud failure instead of a CPU fallback
        with pytest.raises(GmError):
            model(torch.rand(2, 64 * 64 * 3))
        with pytest.raises(GmError):
            model.decoder(torch.randn(2, 20))
        with pytest.raises(GmError):
            model.encoder(torch.rand(2, 64 * 64 * 3))
        with pytest.raises(GmError):
            tr.compute_batch(it[0])
        import copy
        with pytest.raises(GmError):
            copy.deepcopy(model).decoder(torch.randn(2, 20))
