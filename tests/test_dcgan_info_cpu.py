"""InfoGAN on the DCGAN conv path, CPU side: the MI-loss upstream gradient gm_info_loss_rows implements ((softmax - onehot)
inv and 2 (q - c) inv / nc, times LAMBDA; tests/dcgan_info_oracle.py) against float64 autograd of src/info_gan.py's train_Q
expression, alone and composed through the oracle's Q and G, and the surface of the dc_info_gan drop-in.  No GPU needed."""
import inspect

import pytest
import torch

import dcgan_info_oracle as IO
from oracle import dcgan_torch as O


def _noise(n, z, nd, nc, g):
    """compute_noise's layout (src/info_gan.py:311-325): [z N(0,1) | one-hot | nc N(0,1)]"""
    onehot = torch.zeros(n, nd, dtype=torch.float64)
    onehot[range(n), torch.randint(0, nd, (n,), generator=g)] = 1
    return torch.cat([torch.randn(n, z, generator=g, dtype=torch.float64), onehot,
                      torch.randn(n, nc, generator=g, dtype=torch.float64)], 1)


def _nets(hd=8, z=10, nd=7, nc=3, seed=0, wstd=0.05):
    torch.manual_seed(seed)
    G, Qn = O.Generator(hd, z + nd + nc).double(), IO.QNet(hd, nd, nc).double()
    with torch.no_grad():
        for net in (G, Qn):
            for name, p in net.named_parameters():
                if name.split(".")[-2].startswith("l"):
                    p.normal_(0.0, wstd)
    G.train(); Qn.train()
    return G, Qn


@pytest.mark.parametrize("nd,nc,lam", [(10, 10, 1.0), (7, 3, 0.25), (1, 1, 3.0)])
def test_mi_rows_gradient_equals_float64_autograd(nd, nc, lam):
    """the kernel's closed form against autograd of LAMBDA (CE + MSE) on given Q rows (the MSE is a mean over batch x nc)"""
    n, z = 6, 5
    g = torch.Generator().manual_seed(nd * 31 + nc)
    noise = _noise(n, z, nd, nc, g)
    rows = torch.randn(n, nd + nc, generator=g, dtype=torch.float64, requires_grad=True)
    d, c = IO.mi_terms(rows[:, :nd], rows[:, nd:], noise, z)
    ref = torch.autograd.grad(lam * (d + c), rows)[0]
    got = IO.mi_rows_grad(rows.detach(), noise, z, nd, nc, 1.0 / n, lam)
    assert float((got - ref).abs().max() / ref.abs().max()) <= 1e-9


@pytest.mark.parametrize("seed,lam", [(0, 1.0), (1, 0.5)])
def test_mi_step_composition_equals_float64_autograd(seed, lam):
    """the device's order - Q's rows, the closed-form row gradient, Q's backward to G(noise), G's backward - gives every Q
    and G weight gradient of autograd on the reference's MI loss (G_output not detached, src/info_gan.py:286-304)"""
    z, nd, nc, n = 10, 7, 3, 5
    G, Qn = _nets(z=z, nd=nd, nc=nc, seed=seed)
    noise = _noise(n, z, nd, nc, torch.Generator().manual_seed(seed + 7))
    params = list(Qn.parameters()) + list(G.parameters())
    ref = torch.autograd.grad(IO.mi_loss(G, Qn, noise, z, lam), params)
    rows = Qn.rows(G(noise))
    drows = IO.mi_rows_grad(rows.detach(), noise, z, nd, nc, 1.0 / n, lam)
    got = torch.autograd.grad(rows, params, drows, retain_graph=True)
    names = ["Q." + k for k, _ in Qn.named_parameters()] + ["G." + k for k, _ in G.named_parameters()]
    assert len(names) == 11 + 13
    for name, a, b in zip(names, got, ref):
        rel = float((a - b).norm() / b.norm().clamp_min(1e-300))
        assert rel <= 1e-9, (name, rel)
    # both codes matter: without the continuous term the G gradient is a different one
    d_only = IO.mi_rows_grad(rows.detach(), noise, z, nd, nc, 1.0 / n, lam)
    d_only[:, nd:] = 0
    part = torch.autograd.grad(rows, list(G.parameters()), d_only)
    assert float((part[0] - ref[len(list(Qn.parameters()))]).norm()) > 1e-3 * float(ref[len(list(Qn.parameters()))].norm())


def _sig(fn):
    return [(k, v.default) for k, v in inspect.signature(fn).parameters.items()][1:]


def test_dc_info_gan_surface_without_a_gpu():
    import dc_gan
    import dc_info_gan as M
    from gm_b200 import GmError
    E = inspect.Parameter.empty
    # src/info_gan.py:100,130,223,248,269,306,333
    assert _sig(M.DCInfoGAN.__init__) == [("image_size", 64 * 64 * 3), ("hidden_dim", 64), ("z_dim", 100), ("disc_dim", 10),
                                          ("cont_dim", 10), ("output_dim", 1), ("channels", 3)]
    assert _sig(M.DCInfoGANTrainer.train) == [("num_epochs", E), ("G_lr", 2e-4), ("D_lr", 2e-4), ("D_steps", 1)]
    assert _sig(M.DCInfoGANTrainer.train_D) == [("images", E)]
    assert _sig(M.DCInfoGANTrainer.train_G) == [("images", E)]
    assert _sig(M.DCInfoGANTrainer.train_Q) == [("images", E), ("LAMBDA", 1)]
    assert _sig(M.DCInfoGANTrainer.compute_noise) == [("batch_size", E), ("z_dim", E), ("disc_dim", E), ("cont_dim", E), ("c", None)]
    assert _sig(M.DCInfoGANTrainer.generate_images) == [("epoch", E), ("num_outputs", 36), ("save", True), ("c", None)]
    model = M.DCInfoGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100, disc_dim=10, cont_dim=10)
    assert (model.z_dim, model.disc_dim, model.cont_dim, model.image_size, model.hidden_dim, model.shape) == (100, 10, 10, 12288, 16, 64)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCInfoGANTrainer(model, it, it, it)
    assert isinstance(tr, dc_gan.DCGANTrainer) and tr.name == "DCInfoGAN" and tr.variant == "info"
    assert tr.Glosses == [] and tr.Dlosses == [] and tr.MIlosses == []
    for fn in ("save_model", "load_model", "process_batch", "viz_loss"):
        assert callable(getattr(tr, fn))
    sd = model.state_dict()
    bn = lambda pfx, i: ["%s.bn%d.%s" % (pfx, i, k) for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]  # noqa: E731
    ns = dc_gan.DCGAN(hidden_dim=16).state_dict()
    assert [k for k in sd if k.startswith("D.")] == [k for k in ns if k.startswith("D.")]
    assert [k for k in sd if k.startswith("G.")] == [k for k in ns if k.startswith("G.")]
    assert [k for k in sd if k.startswith("Q.")] == ["Q.l%d.weight" % i for i in range(1, 6)] + sum((bn("Q", i) for i in (2, 3, 4)), [])
    assert list(sd)[-1].startswith("Q.")                                                # keys G.*, D.*, then Q.*
    shapes = {"G.l1.weight": (120, 128, 4, 4), "G.l2.weight": (128, 64, 4, 4), "D.l1.weight": (16, 3, 4, 4), "D.l5.weight": (1, 128, 4, 4),
              "Q.l1.weight": (16, 3, 4, 4), "Q.l4.weight": (128, 64, 4, 4), "Q.l5.weight": (20, 128, 4, 4), "Q.bn2.weight": (32,),
              "Q.bn4.running_var": (128,)}
    for k, shp in shapes.items():
        assert tuple(sd[k].shape) == shp, k
    assert tuple(M.DCInfoGAN(hidden_dim=16, z_dim=20, disc_dim=7, cont_dim=3).state_dict()["Q.l5.weight"].shape) == (10, 128, 4, 4)
    assert tuple(M.DCInfoGAN(hidden_dim=16, z_dim=20, disc_dim=7, cont_dim=3).state_dict()["G.l1.weight"].shape) == (30, 128, 4, 4)
    # compute_noise: [z | one-hot | continuous] (src/info_gan.py:311-325), c= fixes the category
    torch.manual_seed(0)
    noise = tr.compute_noise(500, 100, 10, 10).cpu()
    assert noise.shape == (500, 120)
    onehot = noise[:, 100:110]
    assert bool(((onehot == 0) | (onehot == 1)).all()) and bool((onehot.sum(1) == 1).all())
    assert len(set(onehot.argmax(1).tolist())) == 10
    assert abs(float(noise[:, :100].std()) - 1) < 0.05 and abs(float(noise[:, 110:].std()) - 1) < 0.05
    fixed = tr.compute_noise(6, 100, 10, 10, c=3).cpu()
    assert bool((fixed[:, 103] == 1).all()) and float(fixed[:, 100:110].sum()) == 6
    with pytest.raises(GmError):
        M.DCInfoGAN(image_size=784)
    with pytest.raises(GmError):
        M.DCInfoGAN(hidden_dim=16, cont_dim=0)
    if not torch.cuda.is_available():   # no GPU: a loud failure instead of a CPU fallback
        with pytest.raises(GmError):
            model.Q(torch.rand(2, 64 * 64 * 3))
        with pytest.raises(GmError):
            model.G(torch.randn(2, 120))
        with pytest.raises(GmError):
            tr.train_Q(torch.rand(2, 64 * 64 * 3))
