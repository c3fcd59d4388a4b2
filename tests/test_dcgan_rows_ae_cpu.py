"""MMGAN, WGAN, LSGAN, f-GAN and the autoencoder on the DCGAN conv path, CPU side: the torch row losses
(tests/dcgan_rows_oracle.py) against oracle/ref_math.py and central differences, the autoencoder step as the device
decomposes it (tests/dcgan_ae_oracle.py) against float64 autograd, and the surface of the dc_mm_gan, dc_w_gan, dc_ls_gan,
dc_f_gan and dc_ae drop-ins.  No GPU needed."""
import inspect

import numpy as np
import pytest
import torch

import dcgan_ae_oracle as AO
import dcgan_rows_oracle as RO
from oracle import ref_math as R

_E = inspect.Parameter.empty


def _scores(n=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (0.05 + 0.9 * torch.rand(n, 1, generator=g, dtype=torch.float64),
            0.05 + 0.9 * torch.rand(n, 1, generator=g, dtype=torch.float64))


@pytest.mark.parametrize("variant", RO.ROW_VARIANTS)
def test_row_losses_equal_ref_math(variant):
    """at LSGAN's defaults the torch rows are ref_math's losses and upstream gradients"""
    dx, dg = _scores()
    L, gx, gg = R.d_loss(variant, dx.numpy(), dg.numpy())
    x, f = dx.clone().requires_grad_(True), dg.clone().requires_grad_(True)
    Lt = RO.d_rows(variant, x, f)
    tx, tf = torch.autograd.grad(Lt, [x, f])
    assert abs(float(Lt.detach()) - L) <= 1e-12 * max(1.0, abs(L))
    assert np.allclose(tx.numpy(), gx, rtol=1e-12, atol=1e-15) and np.allclose(tf.numpy(), gg, rtol=1e-12, atol=1e-15)
    Lg, gg = R.g_loss(variant, dg.numpy())
    f = dg.clone().requires_grad_(True)
    Lt = RO.g_rows(variant, f)
    assert abs(float(Lt.detach()) - Lg) <= 1e-12 * max(1.0, abs(Lg))
    assert np.allclose(torch.autograd.grad(Lt, f)[0].numpy(), gg, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("variant,abc", [(v, (0.0, 1.0, 1.0)) for v in RO.ROW_VARIANTS] + [("ls", (-1.0, 1.0, 0.0)), ("ls", (0.3, 0.8, 0.6))])
def test_row_gradients_equal_central_differences(variant, abc):
    a, b, c = abc
    dx, dg = _scores(seed=1)
    x, f = dx.clone().requires_grad_(True), dg.clone().requires_grad_(True)
    tx, tf = torch.autograd.grad(RO.d_rows(variant, x, f, a, b), [x, f])
    tg = torch.autograd.grad(RO.g_rows(variant, f, c), f)[0]
    h = 1e-6
    for i in range(dx.shape[0]):
        e = torch.zeros_like(dx)
        e[i] = h
        cx = (RO.d_rows(variant, dx + e, dg, a, b) - RO.d_rows(variant, dx - e, dg, a, b)) / (2 * h)
        cf = (RO.d_rows(variant, dx, dg + e, a, b) - RO.d_rows(variant, dx, dg - e, a, b)) / (2 * h)
        cg = (RO.g_rows(variant, dg + e, c) - RO.g_rows(variant, dg - e, c)) / (2 * h)
        for got, want in ((tx[i], cx), (tf[i], cf), (tg[i], cg)):
            assert abs(float(got) - float(want)) <= 1e-7 * max(1.0, abs(float(want))), (variant, i, float(got), float(want))


def test_ls_targets_enter_as_the_reference_writes_them():
    """src/ls_gan.py:192-193,213 at (a, b, c) = (-1, 1, 0)"""
    dx, dg = _scores(seed=2)
    want_d = 0.5 * torch.mean((dx - 1) ** 2) + 0.5 * torch.mean((dg + 1) ** 2)
    assert float(RO.d_rows("ls", dx, dg, -1.0, 1.0)) == pytest.approx(float(want_d), rel=1e-15)
    assert float(RO.g_rows("ls", dg, 0.0)) == pytest.approx(float(0.5 * torch.mean(dg ** 2)), rel=1e-15)


# ------------------------------------------------------------------ the autoencoder step
def _ae(hd=8, z=6, seed=0, wstd=0.05):
    torch.manual_seed(seed)
    E, G = AO.Encoder(hd, z).double(), AO.Decoder(hd, z).double()
    with torch.no_grad():
        for m in (E, G):
            for name, p in m.named_parameters():
                if name.startswith("l"):
                    p.normal_(0.0, wstd)
    E.train(); G.train()
    return E, G


@pytest.mark.parametrize("zero_unit", [False, True])
def test_ae_step_decomposition_equals_float64_autograd(zero_unit):
    """the device's decomposition of compute_batch + backward (relu code, SSE through the sigmoid, dz, dh = dz 1[h > 0])
    against autograd of the reference's expression; zero_unit zeroes one head row so that h == 0 exactly for every image
    (torch's relu backward gives 0 there, and so does dlatent)"""
    E, G = _ae()
    if zero_unit:
        with torch.no_grad():
            E.l5.weight[2].zero_()
    g = torch.Generator().manual_seed(3)
    x = torch.rand(5, 3 * 4096, generator=g, dtype=torch.float64)
    st = AO.step(E, G, x)
    assert bool((st["code"] == 0).any()) and bool((st["code"] > 0).any())        # both sides of the kink are exercised
    if zero_unit:
        assert bool((st["h"][:, 2] == 0).all()) and bool((st["dh"][:, 2] == 0).all())
    loss = AO.compute_batch(E, G, x)
    params = list(E.parameters()) + list(G.parameters())
    ref = torch.autograd.grad(loss, params)
    assert abs(float(st["loss"] - loss)) <= 1e-12 * float(loss)
    names = ["D." + k for k, _ in E.named_parameters()] + ["G." + k for k, _ in G.named_parameters()]
    for name, r in zip(names, ref):
        got = st["grads"][name]
        rel = float((got - r).norm() / r.norm().clamp_min(1e-300))
        assert rel <= 1e-9, (name, rel)
    assert torch.equal(st["code"], torch.relu(E.head(x)).detach())


# ------------------------------------------------------------------ drop-in surfaces (src/*.py signatures)
def _sig(fn):
    return [(k, v.default) for k, v in inspect.signature(fn).parameters.items()][1:]


def _gan(modname, model_name, trainer_name, variant):
    import dc_gan
    from gm_b200 import GmError
    M = __import__(modname)
    Model, Trainer = getattr(M, model_name), getattr(M, trainer_name)
    model = Model(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = Trainer(model, it, it, it)
    assert isinstance(tr, dc_gan.DCGANTrainer) and tr.name == model_name and tr.variant == variant
    assert list(model.state_dict()) == list(dc_gan.DCGAN(hidden_dim=16).state_dict())
    assert isinstance(model.D, dc_gan.Discriminator) and model.D.out_act == "sigmoid" and M.Generator is dc_gan.Generator
    for fn in ("generate_images", "save_model", "load_model", "compute_noise", "process_batch", "viz_loss"):
        assert callable(getattr(tr, fn))
    with pytest.raises(GmError):
        Model(image_size=784)
    if not torch.cuda.is_available():
        with pytest.raises(GmError):
            model.G(torch.randn(2, 100))
    return M, tr


def test_dc_mm_gan_surface_without_a_gpu():
    M, _ = _gan("dc_mm_gan", "DCMMGAN", "DCMMGANTrainer", "mm")
    # src/mm_gan.py:97,195,220
    assert _sig(M.DCMMGANTrainer.train) == [("num_epochs", _E), ("G_lr", 2e-4), ("D_lr", 2e-4), ("D_steps", 1), ("G_init", 5)]
    assert _sig(M.DCMMGANTrainer.train_D) == [("images", _E)] and _sig(M.DCMMGANTrainer.train_G) == [("images", _E)]


def test_dc_w_gan_surface_without_a_gpu():
    M, tr = _gan("dc_w_gan", "DCWGAN", "DCWGANTrainer", "w")
    # src/w_gan.py:105,190,212,241
    assert _sig(M.DCWGANTrainer.train) == [("num_epochs", _E), ("G_lr", 5e-5), ("D_lr", 5e-5), ("D_steps", 5), ("clip", 0.01)]
    assert _sig(M.DCWGANTrainer.train_D) == [("images", _E)] and _sig(M.DCWGANTrainer.clip_D_weights) == [("clip", _E)]
    # clip_D_weights before any engine exists clamps the modules' parameters, BatchNorm's included
    with torch.no_grad():
        for p in tr.model.D.parameters():
            p.normal_(0.0, 1.0)
    tr.clip_D_weights(0.01)
    assert all(float(p.abs().max()) <= 0.01 for p in tr.model.D.parameters())
    assert float(tr.model.G.l1.weight.abs().max()) > 0.01 and tr._dirty


def test_dc_ls_gan_surface_without_a_gpu():
    M, _ = _gan("dc_ls_gan", "DCLSGAN", "DCLSGANTrainer", "ls")
    # src/ls_gan.py:95,173,197
    assert _sig(M.DCLSGANTrainer.train) == [("num_epochs", _E), ("G_lr", 1e-4), ("D_lr", 1e-4), ("D_steps", 1)]
    assert _sig(M.DCLSGANTrainer.train_D) == [("images", _E), ("a", 0), ("b", 1)]
    assert _sig(M.DCLSGANTrainer.train_G) == [("images", _E), ("c", 1)]
    assert M.DCLSGANTrainer.train_D._gm_builtin and M.DCLSGANTrainer.train_G._gm_builtin


def test_dc_f_gan_surface_without_a_gpu():
    import f_gan
    M, tr = _gan("dc_f_gan", "DCfGAN", "DCfGANTrainer", "f_jensen_shannon")
    # src/f_gan.py:162
    assert _sig(M.DCfGANTrainer.train) == [("num_epochs", _E), ("method", _E), ("G_lr", 1e-4), ("D_lr", 1e-4), ("D_steps", 1)]
    assert M.Divergence is f_gan.Divergence
    tr._set_method("Pearson ")                      # no engine yet: only the variant changes
    assert tr.variant == "f_pearson" and tr._engine is None and tr.loss_fnc.method == "pearson"
    with pytest.raises(AssertionError):
        tr._set_method("kl")


def test_dc_ae_surface_without_a_gpu():
    import dc_ae
    import dc_vae
    from gm_b200 import GmError
    # src/ae.py:58,87
    assert _sig(dc_ae.DCAutoencoder.__init__) == [("image_size", 64 * 64 * 3), ("hidden_dim", 64), ("z_dim", 32), ("channels", 3)]
    assert _sig(dc_ae.DCAutoencoderTrainer.train) == [("num_epochs", _E), ("lr", 1e-3), ("weight_decay", 1e-5)]
    for fn in ("compute_batch", "evaluate", "reconstruct_images", "viz_loss", "save_model", "load_model"):
        assert callable(getattr(dc_ae.DCAutoencoderTrainer, fn))
    model = dc_ae.DCAutoencoder(hidden_dim=16)
    sd = model.state_dict()
    assert [k for k in sd if k.startswith("encoder.") and k.endswith("weight")] == \
        ["encoder.l%d.weight" % i for i in range(1, 6)] + ["encoder.bn%d.weight" % i for i in range(2, 5)]
    assert sd["encoder.l5.weight"].shape == (32, 128, 4, 4) and sd["decoder.l1.weight"].shape == (32, 128, 4, 4)
    assert [k for k in sd if k.startswith("decoder.")] == [k for k in dc_vae.DCVAE(hidden_dim=16, z_dim=32).state_dict()
                                                          if k.startswith("decoder.")]
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = dc_ae.DCAutoencoderTrainer(model, it, it, it)
    assert tr.name == "DCAutoencoder" and tr.recon_loss == [] and tr.best_val_loss == 1e10
    with pytest.raises(GmError):
        dc_ae.DCAutoencoder(image_size=784)
    if not torch.cuda.is_available():
        with pytest.raises(GmError):
            model(torch.zeros(2, 3 * 4096))
