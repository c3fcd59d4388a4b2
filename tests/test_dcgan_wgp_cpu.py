"""WGAN-GP on the DCGAN conv path, CPU side: the closed-form double backward of the batch-norm-free critic
(oracle/dcgan_torch.py, the five steps the CUDA path runs) against autograd's double backward in float64, and the
surface of the dc_w_gp_gan drop-in.  No GPU needed."""
import inspect

import pytest
import torch

from oracle import dcgan_torch as O


def _critic(out_act, sign, hd=8, seed=0):
    torch.manual_seed(seed)
    D = O.Critic(hd, 3, out_act).double()
    with torch.no_grad():
        for l in D.layers():
            l.weight.normal_(0.0, 0.02)
        D.l5.weight.abs_().mul_(sign)
    return D


def _batch(n=5, seed=1):
    g = torch.Generator().manual_seed(seed)
    real = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    fake = torch.rand(n, 3 * 64 * 64, generator=g, dtype=torch.float64)
    eps = torch.rand(n, generator=g, dtype=torch.float64)
    return real, fake, eps


def _rows_with_live_and_dead(D, real, fake, eps):
    """x_hat rows whose logit is positive (live) and negative (dead): a relu critic must be tested on both"""
    return O.Critic.trace(D, O.interpolate(real, fake, eps))[0]


def _mixed_case(out_act):
    """a batch whose x_hat logits have both signs: non-negative images under an all-positive (or all-negative) last layer
    give logits of one sign only, so the case is built with a zero-mean shift of the images"""
    D = _critic(out_act, 1.0)
    real, fake, eps = _batch()
    real, fake = real - 0.5, fake - 0.5
    with torch.no_grad():                   # fix the sign of the last layer per output position so the logits straddle 0
        D.l5.weight[..., :2, :] *= -1
    s = _rows_with_live_and_dead(D, real, fake, eps)
    if not (bool((s > 0).any()) and bool((s < 0).any())):
        # shift row by row: images with a positive / negative offset push the logit to either side
        real = real + torch.linspace(-0.5, 0.5, real.shape[0], dtype=real.dtype).view(-1, 1)
        fake = fake + torch.linspace(-0.5, 0.5, real.shape[0], dtype=real.dtype).view(-1, 1)
        s = _rows_with_live_and_dead(D, real, fake, eps)
    return D, real, fake, eps, s


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_closed_form_penalty_gradient_equals_autograd_double_backward(out_act):
    D, real, fake, eps, s = _mixed_case(out_act)
    assert bool((s > 0).any()) and bool((s < 0).any()), s          # live and dead rows in the same batch
    xh = O.interpolate(real, fake, eps)
    cf = O.closed_form_d_step(D, real, fake, xh, lam=10.0)
    ag = O.autograd_d_step(D, real, fake, xh, lam=10.0)
    assert abs(float(cf["loss"] - ag["loss"])) <= 1e-9 * max(1.0, abs(float(ag["loss"])))
    assert abs(float(cf["gp"] - ag["gp"])) <= 1e-9 * abs(float(ag["gp"]))
    for l, (a, b) in enumerate(zip(cf["grads"], ag["grads"])):
        rel = float((a - b).norm() / b.norm())
        assert rel <= 1e-6, (l, rel)
    if out_act == "relu":
        dead = s <= 0
        assert torch.equal(cf["norms"][dead], torch.zeros(int(dead.sum()), dtype=torch.float64))   # GP = lambda, no gradient
        assert bool((cf["norms"][~dead] > 0).all())
        assert bool((cf["r"].reshape(s.shape[0], -1)[dead] == 0).all())


def test_dead_relu_batch_has_penalty_lambda_and_only_the_w_gradient():
    """every x_hat row dead (s < 0 for non-negative images under a negative last layer): GP = lambda exactly and the
    penalty adds nothing to the gradient"""
    D = _critic("relu", -1.0)
    real, fake, eps = _batch()
    s = _rows_with_live_and_dead(D, real, fake, eps)
    assert bool((s < 0).all())
    xh = O.interpolate(real, fake, eps)
    cf = O.closed_form_d_step(D, real, fake, xh, lam=10.0)
    no_gp = O.closed_form_d_step(D, real, fake, xh, lam=0.0)
    assert float(cf["gp"]) == 10.0
    for a, b in zip(cf["grads"], no_gp["grads"]):
        assert torch.equal(a, b)


def test_split_batch_sums_to_the_full_batch():
    """inv_global_batch scaling: the gradient of 2n images is the sum of two n-image halves at inv = 1 / (2n)"""
    D, real, fake, eps, _ = _mixed_case("relu")
    real, fake, eps = torch.cat([real, real.flip(0)]), torch.cat([fake, fake.flip(0)]), torch.cat([eps, eps.flip(0) * 0.5])
    n = real.shape[0] // 2
    xh = O.interpolate(real, fake, eps)
    full = O.closed_form_d_step(D, real, fake, xh)
    a = O.closed_form_d_step(D, real[:n], fake[:n], xh[:n], inv=1.0 / (2 * n))
    b = O.closed_form_d_step(D, real[n:], fake[n:], xh[n:], inv=1.0 / (2 * n))
    for f, x, y in zip(full["grads"], a["grads"], b["grads"]):
        assert float((f - (x + y)).norm() / f.norm()) < 1e-12


def test_dc_w_gp_gan_surface_without_a_gpu():
    import dc_gan
    import dc_w_gp_gan as M
    from gm_b200 import GmError
    model = M.DCWGPGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    sd = model.state_dict()
    assert not any(k.startswith("D.bn") for k in sd), [k for k in sd if k.startswith("D.")]
    assert [k for k in sd if k.startswith("D.")] == ["D.l%d.weight" % i for i in range(1, 6)]
    assert sd["D.l1.weight"].shape == (16, 3, 4, 4) and sd["D.l5.weight"].shape == (1, 128, 4, 4)
    assert sd["G.l1.weight"].shape == (100, 128, 4, 4) and "G.bn1.running_mean" in sd
    assert model.D.out_act == "relu" and M.Discriminator(64 * 64 * 3, 16, out_act="none").out_act == "none"
    assert M.Generator is dc_gan.Generator
    assert (model.z_dim, model.image_size, model.hidden_dim, model.shape) == (100, 12288, 16, 64)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCWGPGANTrainer(model, it, it, it)
    assert isinstance(tr, dc_gan.DCGANTrainer) and tr.name == "DCWGPGAN" and tr.variant == "wgp"
    # signatures and defaults of src/w_gp_gan.py:96,177,222
    sig = inspect.signature(M.DCWGPGANTrainer.train).parameters
    assert [(k, v.default) for k, v in sig.items()][1:] == [("num_epochs", inspect.Parameter.empty), ("G_lr", 1e-4), ("D_lr", 1e-4),
                                                            ("D_steps", 5)]
    assert [(k, v.default) for k, v in inspect.signature(M.DCWGPGANTrainer.train_D).parameters.items()][1:] == \
        [("images", inspect.Parameter.empty), ("LAMBDA", 10)]
    assert list(inspect.signature(M.DCWGPGANTrainer.train_G).parameters)[1:] == ["images"]
    for name in ("generate_images", "save_model", "load_model", "compute_noise", "process_batch", "viz_loss"):
        assert callable(getattr(tr, name))
    if not torch.cuda.is_available():   # no GPU: a loud failure instead of a CPU fallback
        with pytest.raises(GmError):
            model.G(torch.randn(2, 100))
        with pytest.raises(GmError):
            tr.train_D(torch.zeros(2, 3 * 64 * 64))
    with pytest.raises(GmError):
        M.DCWGPGAN(image_size=784)
    with pytest.raises(GmError):
        M.Discriminator(64 * 64 * 3, 16, out_act="sigmoid")
