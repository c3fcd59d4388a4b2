"""BEGAN on the DCGAN conv path, CPU side: the G-step gradient decomposition the device runs (dL/dG(z) = T - sign(r - G(z))/B,
T through the autoencoder; tests/dcgan_began_oracle.py) against float64 autograd of src/be_gan.py's G loss, and the surface
of the dc_be_gan drop-in.  No GPU needed."""
import inspect

import pytest
import torch

import dcgan_began_oracle as BO
from oracle import dcgan_torch as O


def _nets(hd=8, e=12, z=10, seed=0, wstd=0.05):
    torch.manual_seed(seed)
    G, AE = O.Generator(hd, z).double(), BO.AutoEncoder(hd, e).double()
    with torch.no_grad():
        for net in (G, AE):
            for name, p in net.named_parameters():
                if name.split(".")[-2].startswith("l"):
                    p.normal_(0.0, wstd)
    G.train(); AE.train()
    return G, AE


@pytest.mark.parametrize("seed", [0, 1])
def test_g_step_decomposition_equals_float64_autograd(seed):
    """the device's order - T from the autoencoder's input-gradient chain, minus the direct term through the L1 target -
    gives every G weight gradient of autograd on the reference's G loss (G_output not detached, src/be_gan.py:251-256)"""
    G, AE = _nets(seed=seed)
    n = 5
    z = torch.randn(n, 10, generator=torch.Generator().manual_seed(seed + 7), dtype=torch.float64)
    params = list(G.parameters())
    ref = torch.autograd.grad(BO.g_loss(AE, G, z), params)
    fake = G(z)
    dfake = BO.g_input_grad(AE, fake.detach(), 1.0 / n)
    got = torch.autograd.grad(fake, params, dfake, retain_graph=True)
    for (name, _), a, b in zip(G.named_parameters(), got, ref):
        rel = float((a - b).norm() / b.norm().clamp_min(1e-300))
        assert rel <= 1e-9, (name, rel)
    # both routes matter: without T (the path through D) the gradient is a different one
    direct = torch.autograd.grad(fake, params, -torch.sign(AE(fake.detach()) - fake.detach()) / n)
    assert float((direct[0] - ref[0]).norm()) > 1e-3 * float(ref[0].norm())


def _sig(fn):
    return [(k, v.default) for k, v in inspect.signature(fn).parameters.items()][1:]


def test_dc_be_gan_surface_without_a_gpu():
    import dc_gan
    import dc_be_gan as M
    from gm_b200 import GmError
    E = inspect.Parameter.empty
    # src/be_gan.py:109-110,212,240
    assert _sig(M.DCBEGANTrainer.train) == [("num_epochs", E), ("G_lr", 1e-4), ("D_lr", 1e-4), ("D_steps", 1), ("GAMMA", 0.50),
                                            ("LAMBDA", 1e-3), ("K", 0.00)]
    assert _sig(M.DCBEGANTrainer.train_D) == [("images", E), ("K", E)]
    assert _sig(M.DCBEGANTrainer.train_G) == [("images", E)]
    model = M.DCBEGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    assert (model.z_dim, model.image_size, model.hidden_dim, model.shape) == (100, 12288, 16, 64)
    assert model.D.embed_dim == 100 and M.DCBEGAN(hidden_dim=16, z_dim=100, embed_dim=64).D.embed_dim == 64
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCBEGANTrainer(model, it, it, it)
    assert isinstance(tr, dc_gan.DCGANTrainer) and tr.name == "DCBEGAN" and tr.variant == "be"
    for fn in ("generate_images", "save_model", "load_model", "compute_noise", "process_batch", "viz_loss"):
        assert callable(getattr(tr, fn))
    sd = model.state_dict()
    enc = ["D.encoder.l%d.weight" % i for i in range(1, 6)]
    dec = ["D.decoder.l%d.weight" % i for i in range(1, 6)]
    bn = lambda pfx, i: ["%s.bn%d.%s" % (pfx, i, k) for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]  # noqa: E731
    want = enc + sum((bn("D.encoder", i) for i in (2, 3, 4)), []) + dec + sum((bn("D.decoder", i) for i in (1, 2, 3, 4)), [])
    assert [k for k in sd if k.startswith("D.")] == want
    shapes = {"D.encoder.l1.weight": (16, 3, 4, 4), "D.encoder.l2.weight": (32, 16, 4, 4), "D.encoder.l3.weight": (64, 32, 4, 4),
              "D.encoder.l4.weight": (128, 64, 4, 4), "D.encoder.l5.weight": (100, 128, 4, 4), "D.encoder.bn2.weight": (32,),
              "D.encoder.bn4.running_var": (128,), "D.decoder.l1.weight": (100, 128, 4, 4), "D.decoder.l2.weight": (128, 64, 4, 4),
              "D.decoder.l3.weight": (64, 32, 4, 4), "D.decoder.l4.weight": (32, 16, 4, 4), "D.decoder.l5.weight": (16, 3, 4, 4),
              "D.decoder.bn1.weight": (128,), "D.decoder.bn4.bias": (16,)}
    for k, shp in shapes.items():
        assert tuple(sd[k].shape) == shp, k
    # the DCGAN generator
    assert [k for k in sd if k.startswith("G.")] == [k for k in dc_gan.DCGAN(hidden_dim=16).state_dict() if k.startswith("G.")]
    with pytest.raises(GmError):
        M.DCBEGAN(image_size=784)
    if not torch.cuda.is_available():   # no GPU: a loud failure instead of a CPU fallback
        with pytest.raises(GmError):
            model.D(torch.rand(2, 64 * 64 * 3))
        with pytest.raises(GmError):
            model.G(torch.randn(2, 100))
        with pytest.raises(GmError):
            tr.train_D(torch.rand(2, 64 * 64 * 3), 0.0)
