"""DRAGAN, RaNSGAN and Fisher GAN on the DCGAN conv path, CPU side: the closed-form DRAGAN D gradient (tangent seed r,
shared weight-gradient step; oracle/dcgan_torch.py) against autograd's double backward in float64, and the surface of
the dc_dra_gan, dc_ra_gan and dc_fisher_gan drop-ins.  No GPU needed."""
import inspect

import pytest
import torch

from oracle import dcgan_torch as O


def _critic(hd=8, seed=0, wstd=0.05):
    torch.manual_seed(seed)
    D = O.Critic(hd, 3, "sigmoid").double()
    with torch.no_grad():
        for l in D.layers():
            l.weight.normal_(0.0, wstd)
    return D


def _batch(n=5, seed=1, C=1.0):
    g = torch.Generator().manual_seed(seed)
    real = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    fake = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    delta = torch.rand(n, generator=g, dtype=torch.float64)
    u = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    return real, fake, O.make_xhat(real, delta, u, C)


def _compare(D, real, fake, xh, lam, K):
    cf = O.closed_form_d_step(D, real, fake, xh, lam=lam, K=K)
    ag = O.autograd_d_step(D, real, fake, xh, lam=lam, K=K)
    assert abs(float(cf["loss"] - ag["loss"])) <= 1e-9 * max(1.0, abs(float(ag["loss"])))
    assert abs(float(cf["gp"] - ag["gp"])) <= 1e-9 * max(1.0, abs(float(ag["gp"])))
    assert float((cf["norms"] - ag["norms"]).abs().max()) <= 1e-12
    for l, (a, b) in enumerate(zip(cf["grads"], ag["grads"])):
        rel = float((a - b).norm() / b.norm().clamp_min(1e-300))
        assert rel <= 1e-6 or float((a - b).norm()) <= 1e-15, (l, rel)
    return cf, ag


@pytest.mark.parametrize("K", [1.0, 0.5])
def test_closed_form_dragan_gradient_equals_autograd_double_backward(K):
    D = _critic()
    real, fake, xh = _batch()
    cf, _ = _compare(D, real, fake, xh, 10.0, K)
    assert bool((cf["norms"] > 0).all())
    # the penalty contributes to every layer (it is not the NS gradient alone)
    no_gp = O.closed_form_d_step(D, real, fake, xh, lam=0.0, K=K)
    for a, b in zip(cf["grads"], no_gp["grads"]):
        assert float((a - b).norm()) > 1e-6 * float(a.norm())


def test_saturated_row():
    """one x_hat row scaled so that |s| ~ 40 (the critic is positively homogeneous: s(a x) = a s(x)): sigma' ~ 1e-17, its
    ||g|| ~ 0 and its penalty gradient vanishes like autograd's"""
    D = _critic()
    real, fake, xh = _batch()
    s = O.closed_form_d_step(D, real, fake, xh)["s"]
    xh = xh.clone()
    xh[2] *= 40.0 / float(s[2].abs())
    cf, _ = _compare(D, real, fake, xh, 10.0, 1.0)
    assert abs(float(cf["s"][2])) > 39.0 and float(cf["norms"][2]) < 1e-12
    assert float(cf["r"][2].abs().max()) < 1e-12 * float(cf["r"].abs().max())


def test_zero_input_gradient_rows():
    """||J|| = 0 (a zero last layer): the tangent seed is 0 - torch's norm subgradient - and each row adds lam K^2"""
    D = _critic()
    with torch.no_grad():
        D.l5.weight.zero_()
    real, fake, xh = _batch()
    cf, ag = _compare(D, real, fake, xh, 10.0, 0.5)
    assert bool((cf["norms"] == 0).all()) and bool((cf["r"] == 0).all())
    assert abs(float(cf["gp"]) - 10.0 * 0.25) < 1e-12
    no_gp = O.closed_form_d_step(D, real, fake, xh, lam=0.0, K=0.5)
    for a, b in zip(cf["grads"], no_gp["grads"]):
        assert torch.equal(a, b)


def test_split_batch_sums_to_the_full_batch():
    """inv_global_batch scaling with a shared x_hat (std over the global batch): two halves at inv = 1 / (2n) sum to the
    full batch"""
    D = _critic()
    real, fake, xh = _batch(n=6)
    full = O.closed_form_d_step(D, real, fake, xh)
    a = O.closed_form_d_step(D, real[:3], fake[:3], xh[:3], inv=1.0 / 6)
    b = O.closed_form_d_step(D, real[3:], fake[3:], xh[3:], inv=1.0 / 6)
    for f, x, y in zip(full["grads"], a["grads"], b["grads"]):
        assert float((f - (x + y)).norm() / f.norm()) < 1e-12


def _sig(fn):
    return [(k, v.default) for k, v in inspect.signature(fn).parameters.items()][1:]


def _common_surface(M, model_cls, trainer_cls, variant, name):
    import dc_gan
    from gm_b200 import GmError
    model = model_cls(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    assert (model.z_dim, model.image_size, model.hidden_dim, model.shape) == (100, 12288, 16, 64)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = trainer_cls(model, it, it, it)
    assert isinstance(tr, dc_gan.DCGANTrainer) and tr.name == name and tr.variant == variant
    assert list(inspect.signature(trainer_cls.train_G).parameters)[1:] == ["images"]
    for fn in ("generate_images", "save_model", "load_model", "compute_noise", "process_batch", "viz_loss"):
        assert callable(getattr(tr, fn))
    with pytest.raises(GmError):
        model_cls(image_size=784)
    if not torch.cuda.is_available():   # no GPU: a loud failure instead of a CPU fallback
        with pytest.raises(GmError):
            model.G(torch.randn(2, 100))
    return model, tr


def test_dc_dra_gan_surface_without_a_gpu():
    import dc_gan
    import dc_w_gp_gan
    import dc_dra_gan as M
    model, tr = _common_surface(M, M.DCDRAGAN, M.DCDRAGANTrainer, "dra", "DCDRAGAN")
    sd = model.state_dict()
    assert [k for k in sd if k.startswith("D.")] == ["D.l%d.weight" % i for i in range(1, 6)]
    assert sd["D.l1.weight"].shape == (16, 3, 4, 4) and sd["D.l5.weight"].shape == (1, 128, 4, 4)
    assert sd["G.l1.weight"].shape == (100, 128, 4, 4) and "G.bn1.running_mean" in sd
    assert model.D.out_act == "sigmoid" and isinstance(model.D, dc_w_gp_gan.Discriminator) and M.Generator is dc_gan.Generator
    # src/dra_gan.py:94,174
    assert _sig(M.DCDRAGANTrainer.train) == [("num_epochs", inspect.Parameter.empty), ("G_lr", 1e-4), ("D_lr", 1e-4), ("D_steps", 5)]
    assert _sig(M.DCDRAGANTrainer.train_D) == [("images", inspect.Parameter.empty), ("LAMBDA", 10), ("K", 1), ("C", 1)]


@pytest.mark.parametrize("which", ["ra", "fisher"])
def test_dc_ra_and_fisher_gan_surface_without_a_gpu(which):
    import dc_gan
    if which == "ra":
        import dc_ra_gan as M
        model, tr = _common_surface(M, M.DCRaNSGAN, M.DCRaNSGANTrainer, "ra", "DCRaNSGAN")
        # src/ra_gan.py:106
        assert _sig(M.DCRaNSGANTrainer.train) == [("num_epochs", inspect.Parameter.empty), ("G_lr", 2e-4), ("D_lr", 2e-4), ("D_steps", 1)]
        assert _sig(M.DCRaNSGANTrainer.train_D) == [("images", inspect.Parameter.empty)]
    else:
        import dc_fisher_gan as M
        model, tr = _common_surface(M, M.DCFisherGAN, M.DCFisherGANTrainer, "fisher", "DCFisherGAN")
        # src/fisher_gan.py:101,193
        assert _sig(M.DCFisherGANTrainer.train) == [("num_epochs", inspect.Parameter.empty), ("G_lr", 1e-4), ("D_lr", 1e-4), ("D_steps", 1),
                                                    ("RHO", 1e-6)]
        assert _sig(M.DCFisherGANTrainer.train_D) == [("images", inspect.Parameter.empty)]
    # the batch-norm discriminator of DCGAN
    assert list(model.state_dict()) == list(dc_gan.DCGAN(hidden_dim=16).state_dict())
    assert isinstance(model.D, dc_gan.Discriminator)
