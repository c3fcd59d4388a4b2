"""BIR-VAE on the GPU: the Gaussian-kernel MMD entry against float64, the fused BIR step against the float64 oracle
(tests/bir_vae_oracle.py) with the engine's bf16 storage points, the reference-made golden losses, user-written
compute_batch overrides, refusals and the launch ledger.

Error bound of gm_mmd_gaussian (u = 2^-24).  Each term k_ij = exp(-a_ij), a_ij = |x_i - y_j|^2 / Z^2, is formed in
fp32: the squared distance from Z fp32 differences and FMAs carries a relative error <= (Z + 2) u, the scaling by the
rounded 1/Z^2 adds 2 u, and expf is within 2 ulp, so |dk_ij| <= k_ij ((Z + 4) u a_ij + 2 u).  A tile's terms are summed
in fp32 by each of 8 lanes (at most 16 terms) and combined in a 3-level butterfly: <= 20 u relative to the sum of the
|terms| of the tile; the fp64 sums across tiles and CTAs add nothing measurable (2^-53 scale).  Hence
  |mmd - mmd64| <= lam u sum_terms w k_ij (24 + (Z + 4) a_ij),  w = 1 for the pp and zz sums and 2 for the pz sum,
which must also stay below 1e-5 lam sum_terms w k_ij.  For dz_i the row sums R and sum_j k_ij x_j take the same term
errors and fp32 FMA accumulation (<= 20 u relative to their |terms|), then one fp64 combine and one fp32 rounding:
  |dz_id - dz64_id| <= lam 4/Z^2 u [sum_{j in z} k_ij (24 + (Z + 4) a_ij)(|z_id| + |z_jd|)
                                    + sum_{j in p} k_ij (24 + (Z + 4) a_ij)(|z_id| + |p_jd|)] + u |dz64_id|."""
import numpy as np
import pytest
import torch

import gm_b200
from gm_b200 import GmError
from bir_vae_oracle import bir_vae_step
from inputs import gm_init_weights, load_case, unpack_draws, images_from_bits, params_dict
from make_golden_bir_vae import BIR_SHAPES, SEED
from mlp_harness import VaeReluSides, nrel
from oracle import ref_math as R

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _mmd64(z, p, lam, chunk=256):
    """float64 mmd, dmmd/dz and the bounds of the module docstring, row chunk by row chunk on the GPU"""
    z, p = z.double(), p.double()
    B, Z = z.shape
    tot, absw, bnd = 0.0, 0.0, 0.0
    dz, dzb = torch.zeros_like(z), torch.zeros_like(z)
    for r0 in range(0, B, chunk):
        for rows, first in ((z[r0:r0 + chunk], True), (p[r0:r0 + chunk], False)):
            for cols, w in (((z, 1.0), (p, -2.0)) if first else ((p, 1.0),)):
                a = ((rows[:, None, :] - cols[None, :, :]) ** 2).sum(-1) / (Z * Z)
                k = torch.exp(-a)
                e = k * (24 + (Z + 4) * a)
                tot += w * float(k.sum())
                absw += abs(w) * float(k.sum())
                bnd += abs(w) * float(e.sum())
                if first:
                    s = 1.0 if w > 0 else -1.0
                    # -sum k (z_i - z_j) over z columns, + sum k (z_i - p_j) over p columns
                    dz[r0:r0 + chunk] += -s * (k.sum(1)[:, None] * rows - k @ cols)
                    dzb[r0:r0 + chunk] += e.sum(1)[:, None] * rows.abs() + e @ cols.abs()
    g = lam * 4.0 / (Z * Z)
    return lam * tot, lam * U * bnd, lam * absw, g * dz, g * U * dzb + U * (g * dz).abs()


@pytest.mark.parametrize("Z", [2, 20, 64])
@pytest.mark.parametrize("B", [1, 2, 63, 64, 65, 127, 128, 129, 1000, 4097])
def test_mmd_entry_against_float64(B, Z):
    gen = torch.Generator(device="cuda").manual_seed(B * 100 + Z)
    z = 0.7 * torch.randn(B, Z, device="cuda", generator=gen) + 0.2
    p = torch.randn(B, Z, device="cuda", generator=gen)
    lam = 1000.0
    m, dz = gm_b200.mmd_gaussian(z, p, lam)
    m2, dz2 = gm_b200.mmd_gaussian(z, p, lam)
    assert torch.equal(m, m2) and torch.equal(dz, dz2)                 # fixed reduction order: bitwise repeatable
    m_ng, none = gm_b200.mmd_gaussian(z, p, lam, want_grad=False)
    assert none is None and torch.equal(m_ng, m)
    ref, bound, absw, dref, dbound = _mmd64(z, p, lam)
    err = abs(float(m) - ref)
    assert err <= bound + U * abs(ref), (err, bound)                   # + the final fp32 rounding of mmd
    assert err <= 1e-5 * absw, (err, absw)
    if B == 1:
        k = float(torch.exp(-((z.double() - p.double()) ** 2).sum() / (Z * Z)))
        assert abs(ref - lam * (2 - 2 * k)) <= 1e-12 * lam
    derr = (dz.double() - dref).abs()
    assert bool((derr <= dbound).all()), float((derr / dbound.clamp_min(1e-300)).max())


def _weights(X, H, Z, seed):
    shapes = [("encoder.linear", (H, X)), ("encoder.mu", (Z, H)), ("decoder.linear", (H, Z)), ("decoder.recon", (X, H))]
    W = gm_init_weights(shapes, seed)
    return {k + s: v for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))}


GEOMS = [(784, 400, 20), (16, 16, 1), (208, 208, 32), (1024, 432, 2)]


@pytest.mark.parametrize("geom", GEOMS, ids=["%dx%dx%d" % g for g in GEOMS])
def test_fused_step_against_the_oracle(geom):
    X, H, Z = geom
    eng = gm_b200.BirVaeEngine(X, H, Z, eps_std=1 / 4 ** (13.3 / Z), max_batch=320)
    W = _weights(X, H, Z, 77 + Z)
    eng.load(W)
    rng = np.random.default_rng(X + H + Z)
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    for b in (1, 65, 300):
        x = (rng.random((b, X)) < 0.13).astype(np.float32)
        eps = (eng.eps_std * rng.standard_normal((b, Z))).astype(np.float32)
        prior = rng.standard_normal((b, Z)).astype(np.float32)
        P = {k: v.double().cpu().numpy() for k, v in eng.views().items()}
        ls = eng.grad(torch.from_numpy(x).cuda(), eps=torch.from_numpy(eps).cuda(), prior=torch.from_numpy(prior).cuda(),
                      lam=1000.0).cpu().numpy()
        sides = VaeReluSides(eng)
        mse, m, g, fw = bir_vae_step(P, x.astype(np.float64), eps.astype(np.float64), prior.astype(np.float64), 1000.0,
                                     q=R.bf16_points, relu=sides)
        assert abs(ls[0] - mse) <= 1e-3 * mse, (b, ls[0], mse)
        zd, pd = eng.last_latent(b)
        _, _, absw, _, _ = _mmd64(zd, pd, 1000.0)
        assert abs(ls[1] - m) <= 1e-3 * absw, (b, ls[1], m, absw)
        assert nrel(zd.cpu().numpy(), fw["z"]) < 1e-4
        gv = {k: v.cpu().numpy() for k, v in eng.views(eng.grads).items()}
        for k in g:
            assert nrel(gv[k], g[k]) < 3e-3, (b, k, nrel(gv[k], g[k]))
        # one Adam step (coupled weight decay) on the device's own gradient
        before = {k: v.clone() for k, v in eng.views().items()}
        eng.apply(hp)
        t = eng.steps
        for k, p0 in before.items():
            p0, gk = p0.double(), eng.views(eng.grads)[k].double()
            gk = gk + 1e-5 * p0
            mm, vv = 0.1 * gk, 0.001 * gk * gk
            upd = 1e-3 / (1 - 0.9 ** t) * mm / ((vv / (1 - 0.999 ** t)).sqrt() + 1e-8)
            if t == 1:
                assert nrel((p0 - eng.views()[k].double()).cpu().numpy(), upd.cpu().numpy()) < 1e-4, k
        eng.reset_optimizer()


def test_golden_losses_on_the_host_draw_path():
    """the reference's own three train() steps (tests/golden/bir_vae.npz) with its recorded eps and prior draws"""
    fx = load_case("bir_vae")
    X, H, Z = 784, 400, 20
    eng = gm_b200.BirVaeEngine(X, H, Z, eps_std=1 / 4 ** (13.3 / Z), max_batch=64)
    W = gm_init_weights(BIR_SHAPES, SEED)
    eng.load({k + s: v for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))})
    x = torch.from_numpy(images_from_bits(fx)).cuda()
    priors = unpack_draws(fx)
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    mse, mmd = [], []
    for s in range(len(fx["recon_loss"])):
        ls = eng.grad(x, eps=torch.from_numpy(fx["eps"][s]).cuda(), prior=torch.from_numpy(priors[s]).cuda()).cpu().numpy()
        eng.apply(hp)
        mse.append(ls[0])
        mmd.append(ls[1])
    np.testing.assert_allclose(mse, fx["recon_loss"], rtol=2e-3)
    np.testing.assert_allclose(mmd, fx["mmd_loss"], rtol=2e-2)     # lam = 1000 times a difference of B^2-term sums


def _loader(n=130, bs=65, seed=0):
    g = torch.Generator().manual_seed(seed)
    imgs = (torch.rand(n, 1, 28, 28, generator=g) < 0.13).float()
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(n)), batch_size=bs)


def _reference_body(LAMBDA):
    """the reference's compute_batch body (src/bir_vae.py:178-188) with another default LAMBDA"""
    from bir_vae import to_cuda

    def compute_batch(self, batch, LAMBDA=LAMBDA):
        images, _ = batch
        images = to_cuda(images.view(images.shape[0], -1))
        outputs, z = self.model(images)
        mse_loss = torch.sum((images - outputs) ** 2)
        mmd_loss = LAMBDA * self.maximum_mean_discrepancy(z)
        return mse_loss, mmd_loss
    return compute_batch


def _grads_of(trainer, batch, np_seed, torch_seed):
    for p in trainer.model.parameters():
        p.grad = None
    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    mse, mmd = trainer.compute_batch(batch)
    (mse + mmd).backward()
    return float(mse), float(mmd), {k: p.grad.detach().double().cpu().numpy() for k, p in trainer.model.named_parameters()}


def test_reference_compute_batch_override_matches_the_fused_step():
    import bir_vae
    loader = _loader()
    batch = next(iter(loader))
    torch.manual_seed(3)
    m1 = bir_vae.BIRVAE(784, 400, 20)
    m2 = bir_vae.BIRVAE(784, 400, 20)
    m2.load_state_dict(m1.state_dict())
    fused = bir_vae.BIRVAETrainer(m1, loader, loader, loader)
    Custom = type("Custom", (bir_vae.BIRVAETrainer,), {"compute_batch": _reference_body(1000.)})
    custom = Custom(m2, loader, loader, loader)
    a = _grads_of(fused, batch, 11, 12)
    b = _grads_of(custom, batch, 11, 12)
    assert abs(a[0] - b[0]) <= 1e-3 * a[0] and abs(a[1] - b[1]) <= 1e-3 * max(abs(a[1]), 1.0)
    for k in a[2]:
        assert nrel(b[2][k], a[2][k]) < 1e-2, (k, nrel(b[2][k], a[2][k]))


def test_lambda_10_override_matches_float64():
    import bir_vae
    loader = _loader()
    batch = next(iter(loader))
    torch.manual_seed(4)
    model = bir_vae.BIRVAE(784, 400, 20)
    P = {k: v.detach().double().numpy() for k, v in model.state_dict().items()}
    Custom = type("Custom", (bir_vae.BIRVAETrainer,), {"compute_batch": _reference_body(10.)})
    tr = Custom(model, loader, loader, loader)
    mse, mmd, g = _grads_of(tr, batch, 21, 22)
    np.random.seed(21)
    eps = np.random.normal(loc=0.0, scale=model.set_var, size=(65, 20)).astype(np.float32).astype(np.float64)
    torch.manual_seed(22)
    prior = torch.randn(65, 20).double().numpy()
    x = batch[0].view(65, -1).double().numpy()
    mse_o, mmd_o, g_o, _ = bir_vae_step(P, x, eps, prior, 10.0)
    assert abs(mse - mse_o) <= 1e-2 * mse_o
    assert abs(mmd - mmd_o) <= 2e-2 * max(abs(mmd_o), 1.0)
    for k in g_o:
        assert nrel(g[k], g_o[k]) < 3e-2, (k, nrel(g[k], g_o[k]))


def test_maximum_mean_discrepancy_beyond_the_reference_expression():
    """B = 12000, Z = 20: each of the reference's [B, B, Z] fp32 tensors would take 11.5 GB"""
    import bir_vae
    loader = _loader(8, 4)
    tr = bir_vae.BIRVAETrainer(bir_vae.BIRVAE(784, 32, 20), loader, loader, loader)
    B, Z = 12000, 20
    assert B * B * Z * 4 > 5e9
    z = (0.5 * torch.randn(B, Z, device="cuda")).requires_grad_(True)
    torch.manual_seed(5)
    m = tr.maximum_mean_discrepancy(z)
    m.backward()
    torch.manual_seed(5)
    p = torch.randn(B, Z).cuda()
    ref, bound, absw, dref, dbound = _mmd64(z.detach(), p, 1.0, chunk=1024)
    assert abs(float(m) - ref) <= bound + U * abs(ref) and abs(float(m) - ref) <= 1e-5 * absw
    assert bool(((z.grad.double() - dref).abs() <= dbound).all())


def test_fused_train_prints_the_epoch_line_and_round_trips(tmp_path, capsys):
    import bir_vae
    loader = _loader(260, 65)
    model = bir_vae.BIRVAE(784, 400, 20, I=13.3)
    tr = bir_vae.BIRVAETrainer(model, loader, loader, loader)
    tr.train(num_epochs=2, lr=1e-3, weight_decay=1e-5)
    out = capsys.readouterr().out
    assert "Epoch[2/2], Total Loss: " in out and ", MSE Loss: " in out and ", MMD Loss: " in out and ", Val Loss: " in out
    assert len(tr.recon_loss) == len(tr.mmd_loss) == 8 and all(np.isfinite(tr.recon_loss + tr.mmd_loss))
    assert tr.recon_loss[-1] < tr.recon_loss[0]
    path = str(tmp_path / "bir.pt")
    tr.save_model(path)
    sd = torch.load(path)
    assert list(sd) == ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.mu.bias",
                        "decoder.linear.weight", "decoder.linear.bias", "decoder.recon.weight", "decoder.recon.bias"]
    tr2 = bir_vae.BIRVAETrainer(bir_vae.BIRVAE(784, 400, 20), loader, loader, loader)
    tr2.load_model(path)
    for k, v in tr2.model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k].cpu())
    tr.device_noise = False                                                    # the reference's host draws
    tr.train(num_epochs=1)
    assert len(tr.recon_loss) == 12 and isinstance(tr.best_model, bir_vae.BIRVAE)
    assert tr.sample_images().shape == (36, 28, 28)
    assert tr.reconstruct_images(loader.dataset.tensors[0][:4], 0).shape == (4, 28, 28)


def _rc(fn, *a):
    from gm_b200._lib import lib
    return getattr(lib(), fn)(*a)


def test_refusals_before_any_launch():
    import ctypes as C
    from gm_b200._lib import ctx, VaeDesc, PRECISIONS
    h = ctx()
    z = torch.zeros(8, 4, device="cuda")
    out = torch.zeros(2, device="cuda")
    vp = C.c_void_p
    n0 = gm_b200.launch_count()
    bad = [(vp(z.data_ptr()), vp(z.data_ptr()), 0, 4), (vp(z.data_ptr()), vp(z.data_ptr()), -3, 4),
           (vp(z.data_ptr()), vp(z.data_ptr()), 8, 0), (vp(z.data_ptr()), vp(z.data_ptr()), 8, 65),
           (None, vp(z.data_ptr()), 8, 4), (vp(z.data_ptr()), None, 8, 4), (vp(z.data_ptr() + 2), vp(z.data_ptr()), 8, 4),
           (vp(z.data_ptr()), vp(z.data_ptr()), 1 << 26, 64)]
    for zz, pp, b, zd in bad:
        assert _rc("gm_mmd_gaussian", h, zz, pp, b, zd, 1.0, vp(out.data_ptr()), None, None) != 0, (b, zd)
    assert _rc("gm_mmd_gaussian", h, vp(z.data_ptr()), vp(z.data_ptr()), 8, 4, 1.0, None, None, None) != 0
    assert _rc("gm_mmd_gaussian", h, vp(z.data_ptr()), vp(z.data_ptr()), 8, 4, 1.0, vp(out.data_ptr()), vp(z.data_ptr() + 1), None) != 0
    assert gm_b200.launch_count() == n0
    with pytest.raises(GmError, match="bf16 only"):
        gm_b200.BirVaeEngine(784, 400, 20, max_batch=8, precision="split")
    with pytest.raises(GmError, match="z_dim <= 32"):
        gm_b200.BirVaeEngine(784, 400, 33, max_batch=8)
    with pytest.raises(GmError, match="eps_std"):
        gm_b200.BirVaeEngine(784, 400, 20, eps_std=float("nan"), max_batch=8)
    bir = gm_b200.BirVaeEngine(784, 400, 20, max_batch=8)
    vae = gm_b200.VaeEngine(784, 400, 20, max_batch=8)
    x = torch.zeros(8, 784, device="cuda")
    n0 = gm_b200.launch_count()
    with pytest.raises(GmError, match="BIR-VAE engine"):
        gm_b200.VaeEngine.grad(bir, x)
    with pytest.raises(GmError, match="BIR-VAE engine"):
        gm_b200.VaeEngine.forward(bir, x, want_losses=True)
    with pytest.raises(GmError, match="not a BIR-VAE engine"):
        gm_b200.BirVaeEngine.grad(vae, x)
    with pytest.raises(GmError, match="not a BIR-VAE engine"):
        gm_b200.BirVaeEngine.forward(vae, x)
    with pytest.raises(GmError, match="batch must be"):
        bir.grad(x, batch=9)
    with pytest.raises(GmError, match="batch must be"):
        bir.grad(x, batch=0)
    with pytest.raises(GmError, match="slot"):
        bir.encoder_forward(5, x)
    assert gm_b200.launch_count() == n0


def test_launch_ledger_names_the_new_kernels():
    eng = gm_b200.BirVaeEngine(784, 400, 20, max_batch=64)
    x = (torch.rand(64, 784, device="cuda") < 0.13).float()
    gm_b200.prof_enable(2)
    try:
        eng.grad(x)
        eng.forward(x, want_losses=True)
        gm_b200.mmd_gaussian(torch.randn(10, 3, device="cuda"), torch.randn(10, 3, device="cuda"))
        torch.cuda.synchronize()
        names = {n: c for n, c, _ in gm_b200.prof_report()}
    finally:
        gm_b200.prof_enable(0)
    for k in ("bir_latent_kernel", "bir_dlatent_kernel", "mmd_tile_kernel<grad>", "mmd_tile_kernel", "mmd_final_kernel"):
        assert names.get(k, 0) >= 1, (k, names)
