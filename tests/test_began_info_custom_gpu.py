"""User-written train_D / train_G / train_Q (README.md:31) on the MLP BEGAN and InfoGAN trainers, on the GPU: BEGAN's
autoencoder D (gm_gan_ae_*) and InfoGAN's Q (gm_gan_q_*) as autograd nodes against the float64 oracle at the bf16 storage
points, the reference's own method bodies as overrides reproducing its golden losses, losses the fused step does not have,
mixed overrides, the error paths, and the launch ledger of the four entries."""
import numpy as np
import pytest
import torch

from inputs import B, BEGAN_SHAPES, INFO_SHAPES, STEPS, gm_init_weights, images_from_bits, load_case, unpack_draws
from mlp_harness import TOL_A, gan_engine, nrel
from oracle import ref_math as R

pytestmark = pytest.mark.gpu

TOL = 1e-3
MAX_BATCH = 320
BATCHES = (1, 65, 300)
# the reference geometry and the smallest / largest ones tests/test_mlp_geometry_gpu.py runs BEGAN and InfoGAN at
BEGAN_GEOMS = [(784, 400, 20), (16, 16, 1), (1024, 432, 447)]
INFO_GEOMS = [(784, 400, 20), (16, 16, 1), (1024, 432, 427)]
AE_NAMES = ["D.encoder.weight", "D.encoder.bias", "D.decoder.weight", "D.decoder.bias"]
Q_NAMES = ["Q.linear.weight", "Q.linear.bias", "Q.inference.weight", "Q.inference.bias"]


def _gid(g):
    return "%dx%dx%d" % g


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _storage_points(near, act):
    """bf16_points, with the hidden units whose float64 pre-activation lies within TOL_A of the ReLU kink taking the side
    the device took (mlp_harness.DeviceReluSides)"""
    def q(name, v):
        if name == "h" and near.any():
            v = v.copy()
            v[near] = np.where(act[near], 1e-30, 0.0)
        return R.bf16_round(v)
    return q


def _info_engine(X, H, z, max_batch=MAX_BATCH):
    import gm_b200
    W = gm_init_weights([("G.linear", (H, z + 20)), ("G.generate", (X, H)), ("D.linear", (H, X)),
                         ("D.discriminator", (1, H)), ("Q.linear", (H, X)), ("Q.inference", (20, H))], 1234)
    eng = gm_b200.InfoGanEngine(X, H, z, 10, 10, max_batch=max_batch)
    eng.load(0, [W["G.linear"][0], W["G.linear"][1], W["G.generate"][0], W["G.generate"][1]])
    eng.load(1, [W["D.linear"][0], W["D.linear"][1], W["D.discriminator"][0], W["D.discriminator"][1]])
    eng.load_q([W["Q.linear"][0], W["Q.linear"][1], W["Q.inference"][0], W["Q.inference"][1]])
    return eng


# ---------------------------------------------------------------- 1 + 2: the nodes against the float64 oracle
@pytest.mark.parametrize("geom", BEGAN_GEOMS, ids=_gid)
def test_autoencoder_entries_match_oracle(geom):
    """recon, every D gradient and dx of gm_gan_ae_forward / _backward with a random upstream against began_ae /
    began_ae_backward (bf16 engines: the entries refuse split precision)"""
    X, H, Z = geom
    eng = gan_engine("began", X, H, Z, max_batch=MAX_BATCH)
    P = {n: _np(v) for n, v in zip(AE_NAMES, eng.views(1))}
    rng = np.random.default_rng([X, H, Z, 5])
    errs, near_units = {}, 0
    for slot, b in zip((0, 1, 0), BATCHES):
        x = rng.random((b, X)).astype(np.float32)               # grey levels, as G(z) feeds D
        recon = eng.ae_forward(slot, torch.from_numpy(x).cuda())
        xq = R.bf16_round(x.astype(np.float64))
        a1 = xq @ R.bf16_round(P["D.encoder.weight"]).T + P["D.encoder.bias"]
        near = np.abs(a1) < TOL_A
        act = eng.debug_read("Aall", slot * MAX_BATCH, b, H).cpu().numpy() > 0
        near_units += int(near.sum())
        q = _storage_points(near, act)
        fw = R.began_ae(P, xq, q)
        errs["b%d_recon" % b] = nrel(_np(recon), fw["r"])
        dr = (rng.standard_normal((b, X)) / b).astype(np.float32)
        flat, dx = eng.ae_backward(slot, torch.from_numpy(dr).cuda(), True)
        go, dxo = R.began_ae_backward(P, fw, dr.astype(np.float64), q, need_dx=True)
        for n, g in zip(AE_NAMES, eng.views(1, flat)):
            errs["b%d_%s" % (b, n)] = nrel(_np(g), go[n])
        errs["b%d_dx" % b] = nrel(_np(dx), dxo)
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (bad, near_units)


@pytest.mark.parametrize("geom", INFO_GEOMS, ids=_gid)
def test_q_entries_match_oracle(geom):
    """codes, every Q gradient and dx of gm_gan_q_forward / _backward with a random upstream against the Q half of
    info_q_step (src/info_gan.py:78-94), float64 at the bf16 storage points"""
    X, H, z = geom
    eng = _info_engine(X, H, z)
    P = {n: _np(v) for n, v in zip(Q_NAMES, eng.q_views())}
    W1, W2 = R.bf16_round(P["Q.linear.weight"]), R.bf16_round(P["Q.inference.weight"])
    rng = np.random.default_rng([X, H, z, 6])
    errs, near_units = {}, 0
    for slot, b in zip((0, 1, 0), BATCHES):
        x = rng.random((b, X)).astype(np.float32)
        codes = eng.q_forward(slot, torch.from_numpy(x).cuda())
        xq = R.bf16_round(x.astype(np.float64))
        a1 = R.linear(xq, W1, P["Q.linear.bias"])
        near = np.abs(a1) < TOL_A
        act = eng.debug_read("HQ%d" % slot, 0, b, H).cpu().numpy() > 0
        near_units += int(near.sum())
        q = _storage_points(near, act)
        hq = q("h", np.maximum(a1, 0))
        inf = R.linear(hq, W2, P["Q.inference.bias"])
        errs["b%d_codes" % b] = nrel(_np(codes), inf)
        dc = (rng.standard_normal((b, 20)) / b).astype(np.float32)
        flat, dx = eng.q_backward(slot, torch.from_numpy(dc).cuda(), True)
        dinf = R.bf16_round(dc.astype(np.float64))
        dhq = R.bf16_round((dinf @ W2) * (hq > 0))
        go = {"Q.inference.weight": dinf.T @ hq, "Q.inference.bias": dinf.sum(0),
              "Q.linear.weight": dhq.T @ xq, "Q.linear.bias": dhq.sum(0)}
        for n, g in zip(Q_NAMES, eng.q_views(flat)):
            errs["b%d_%s" % (b, n)] = nrel(_np(g), go[n])
        errs["b%d_dx" % b] = nrel(_np(dx), dhq @ W1)
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (bad, near_units)


# ---------------------------------------------------------------- 3: the reference's own bodies as overrides
def _load(model, W):
    sd = model.state_dict()
    for k, (w, b) in W.items():
        sd[k + ".weight"], sd[k + ".bias"] = torch.from_numpy(w.copy()), torch.from_numpy(b.copy())
    model.load_state_dict(sd)


def _began_override():
    import be_gan

    class MyBEGANTrainer(be_gan.BEGANTrainer):
        """src/be_gan.py:212-258 typed in verbatim"""

        def train_D(self, images, K):
            DX_reconst = self.model.D(images)
            DX_loss = torch.mean(torch.sum(torch.abs(DX_reconst - images), dim=1))
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            G_output = self.model.G(noise)
            DG_reconst = self.model.D(G_output)
            DG_loss = torch.mean(torch.sum(torch.abs(DG_reconst - G_output), dim=1))
            D_loss = DX_loss - (K * DG_loss)
            return D_loss, DX_loss, DG_loss

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            G_output = self.model.G(noise)
            DG_reconst = self.model.D(G_output)
            G_loss = torch.mean(torch.sum(torch.abs(DG_reconst - G_output), dim=1))
            return G_loss

    return be_gan, MyBEGANTrainer


def _info_override():
    import torch.nn.functional as F
    import info_gan

    class MyInfoGANTrainer(info_gan.InfoGANTrainer):
        """src/info_gan.py:223-304 typed in verbatim"""

        def train_D(self, images):
            DX_score = self.model.D(images)
            noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim)
            G_output = self.model.G(noise)
            DG_score = self.model.D(G_output)
            D_loss = -torch.mean(torch.log(DX_score + 1e-8) + torch.log(1 - DG_score + 1e-8))
            return torch.sum(D_loss)

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim, c=None)
            G_output = self.model.G(noise)
            DG_score = self.model.D(G_output)
            G_loss = -torch.mean(torch.log(DG_score + 1e-8))
            return G_loss

        def train_Q(self, images, LAMBDA=1):
            G_labels = torch.zeros(images.shape[0], 1).cuda()  # noqa: F841  (as in the reference)
            noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim)
            G_output = self.model.G(noise)
            Q_discrete, Q_continuous = self.model.Q(G_output)
            discrete_target = noise[:, self.model.z_dim:self.model.z_dim + self.model.disc_dim]
            disc_loss = F.cross_entropy(Q_discrete, torch.max(discrete_target, 1)[1])
            continuous_target = noise[:, self.model.z_dim + self.model.disc_dim:]
            cont_loss = F.mse_loss(Q_continuous, continuous_target)
            MI_loss = LAMBDA * (disc_loss + cont_loss)
            return MI_loss

    return info_gan, MyInfoGANTrainer


def _trainer(kind, Trainer=None, steps=STEPS):
    """(trainer over the golden images with compute_noise replaying the reference's draws, fixture)"""
    if kind == "began":
        mod, Custom = _began_override()
        fx, W, model = load_case("gan_began"), gm_init_weights(BEGAN_SHAPES, 1234), mod.BEGAN(784, 400, 20)
    else:
        mod, Custom = _info_override()
        fx, W, model = load_case("gan_info"), gm_init_weights(INFO_SHAPES, 1234), mod.InfoGAN(784, 400, 20, 10, 10)
    _load(model, W)
    x = torch.from_numpy(images_from_bits(fx)).view(B, 1, 28, 28)
    it = [(x, torch.zeros(B, dtype=torch.long))] * steps
    tr = (Trainer or Custom)(model, it, it, it, viz=False)
    draws = iter(unpack_draws(fx))
    tr.compute_noise = lambda *a, **k: torch.from_numpy(next(draws)).cuda()
    return tr, fx


def _close(got, ref, what):
    for a, b in zip(got, ref):
        assert abs(a - b) < 2e-3 * max(abs(b), 0.5), (what, got, list(ref))


@pytest.mark.parametrize("kind", ["began", "info"])
def test_reference_bodies_reproduce_the_golden_losses(kind, capsys):
    from gm_b200 import _lib
    tr, fx = _trainer(kind)
    assert tr._has_custom_step()
    _lib.launch_count(reset=True)
    if kind == "began":
        tr.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)
    else:
        tr.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1)
    assert _lib.launch_count() > 20 * STEPS          # the GEMMs / Adam ran in libgm_b200.so, not in torch
    assert len(tr.Dlosses) == STEPS and len(tr.Glosses) == STEPS and tr.num_epochs == 1
    _close(tr.Dlosses, fx["D_loss"], "D_loss")
    _close(tr.Glosses, fx["G_loss"], "G_loss")
    line = capsys.readouterr().out.strip().splitlines()[-1]
    if kind == "began":
        assert line.startswith("Epoch[1/1], G Loss: ") and ", K: " in line and ", Convergence Measure: " in line, line
    else:
        assert len(tr.MIlosses) == STEPS
        _close(tr.MIlosses, fx["MI_loss"], "MI_loss")
        assert line.startswith("Epoch[1/1], G Loss: ") and ", MI Loss: " in line, line


# ---------------------------------------------------------------- 4: losses the fused step does not have
def _bf16(t):
    """a float64 tensor rounded to bf16 where the device stores it; the gradient passes through"""
    return t + (t.to(torch.bfloat16).to(torch.float64) - t).detach()


def _t64(p):
    return p.detach().to(torch.float64).clone().requires_grad_(True)


def test_squared_error_began_train_D_matches_float64_autograd():
    """a BEGAN train_D with squared instead of absolute reconstruction error: one call + backward against float64
    torch autograd of the same expression, at the same weights and draws, with operands at the bf16 storage points"""
    import be_gan

    class L2BEGAN(be_gan.BEGANTrainer):
        def train_D(self, images, K):
            DX_loss = torch.mean(torch.sum((self.model.D(images) - images) ** 2, dim=1))
            G_output = self.model.G(self.compute_noise(images.shape[0], self.model.z_dim))
            DG_loss = torch.mean(torch.sum((self.model.D(G_output) - G_output) ** 2, dim=1))
            return DX_loss - K * DG_loss, DX_loss, DG_loss

    tr, fx = _trainer("began", L2BEGAN)
    noise = unpack_draws(fx)[0]
    tr._ensure_engine(B)
    images = tr.process_batch(tr.train_iter)
    K = 0.3
    D_loss, _, _ = tr.train_D(images, K)
    D_loss.backward()
    m = tr.model
    G = [_t64(p) for p in m.G.parameters()]
    D = [_t64(p) for p in m.D.parameters()]

    def ae(x):
        h = _bf16(torch.relu(_bf16(x) @ _bf16(D[0]).T + D[1]))
        return h @ _bf16(D[2]).T + D[3]
    x = images.to(torch.float64)
    z = torch.from_numpy(noise).cuda().to(torch.float64)
    fake = _bf16(torch.sigmoid(_bf16(torch.relu(_bf16(z) @ _bf16(G[0]).T + G[1])) @ _bf16(G[2]).T + G[3]))
    ref = torch.mean(torch.sum((ae(x) - x) ** 2, dim=1)) - K * torch.mean(torch.sum((ae(fake) - fake) ** 2, dim=1))
    ref.backward()
    assert abs(D_loss.item() - ref.item()) <= 1e-3 * abs(ref.item())
    for p, r in zip(m.D.parameters(), D):
        assert nrel(_np(p.grad), _np(r.grad)) <= 1e-2, (p.shape, nrel(_np(p.grad), _np(r.grad)))
    for p, r in zip(m.G.parameters(), G):
        assert nrel(_np(p.grad), _np(r.grad)) <= 3e-2, (p.shape, nrel(_np(p.grad), _np(r.grad)))


def test_infogan_train_Q_with_lambda_half_matches_float64_autograd():
    """an InfoGAN train_Q with LAMBDA = 0.5 (the fused MI step is built for 1): one call + backward against float64
    torch autograd of the same expression at the same weights and draws"""
    import torch.nn.functional as F
    info_gan, Custom = _info_override()

    class HalfQ(Custom):
        def train_Q(self, images, LAMBDA=0.5):
            return Custom.train_Q(self, images, LAMBDA)

    tr, fx = _trainer("info", HalfQ)
    noise = unpack_draws(fx)[0]                       # train_Q makes the first draw here
    tr._ensure_engine(B)
    images = tr.process_batch(tr.train_iter)
    MI_loss = tr.train_Q(images)
    MI_loss.backward()
    m = tr.model
    G = [_t64(p) for p in m.G.parameters()]
    Q = [_t64(p) for p in m.Q.parameters()]
    z = torch.from_numpy(noise).cuda().to(torch.float64)
    fake = _bf16(torch.sigmoid(_bf16(torch.relu(_bf16(z) @ _bf16(G[0]).T + G[1])) @ _bf16(G[2]).T + G[3]))
    inf = _bf16(torch.relu(fake @ _bf16(Q[0]).T + Q[1])) @ _bf16(Q[2]).T + Q[3]
    ref = 0.5 * (F.cross_entropy(inf[:, :10], torch.max(z[:, 20:30], 1)[1]) + F.mse_loss(inf[:, 10:], z[:, 30:]))
    ref.backward()
    assert abs(MI_loss.item() - ref.item()) <= 1e-3 * abs(ref.item())
    for p, r in zip(m.Q.parameters(), Q):
        assert nrel(_np(p.grad), _np(r.grad)) <= 1e-2, (p.shape, nrel(_np(p.grad), _np(r.grad)))
    for p, r in zip(m.G.parameters(), G):
        assert nrel(_np(p.grad), _np(r.grad)) <= 3e-2, (p.shape, nrel(_np(p.grad), _np(r.grad)))


# ---------------------------------------------------------------- 5: mixed overrides
@pytest.mark.parametrize("kind", ["began", "info"])
def test_only_train_G_overridden(kind):
    """train_G alone overridden: train() runs the reference loop, the built-in train_D (and train_Q) hand their fused
    gradients to FusedAdam, and every loss is finite"""
    mod, Custom = _began_override() if kind == "began" else _info_override()
    Base = mod.BEGANTrainer if kind == "began" else mod.InfoGANTrainer
    OnlyG = type("OnlyG", (Base,), {"train_G": Custom.train_G})
    tr, _ = _trainer(kind, OnlyG)
    assert tr._has_custom_step()
    tr._ensure_engine(B)                              # the parameters become views of the engine's masters
    d0 = [p.detach().clone() for p in tr.model.D.parameters()]
    if kind == "began":
        tr.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)
    else:
        q0 = [p.detach().clone() for p in tr.model.Q.parameters()]
        tr.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1)
        assert len(tr.MIlosses) == STEPS and np.isfinite(tr.MIlosses).all()
        assert all(not torch.equal(a, b) for a, b in zip(q0, tr.model.Q.parameters()))     # the built-in train_Q trained Q
    assert len(tr.Dlosses) == STEPS and np.isfinite(tr.Dlosses).all() and np.isfinite(tr.Glosses).all()
    assert all(not torch.equal(a, b) for a, b in zip(d0, tr.model.D.parameters()))         # the built-in train_D trained D


# ---------------------------------------------------------------- 6: error paths
def _refused(fn, what):
    from gm_b200 import GmError, _lib
    n0 = _lib.launch_count()
    with pytest.raises(GmError, match=what):
        fn()
    assert _lib.launch_count() == n0


def test_overwritten_calls_and_double_backward_raise():
    tr, _ = _trainer("began")
    x = torch.rand(8, 784, device="cuda")
    D = tr.model.D
    r0 = D(x)
    D(x), D(x)                                        # two later calls take both row regions
    with pytest.raises(RuntimeError, match="overwritten"):
        r0.sum().backward()
    with pytest.raises(RuntimeError, match="double backward"):
        D(x).sum().backward(create_graph=True)
    tri, _ = _trainer("info")
    tri._ensure_engine(B)
    Qm = tri.model.Q
    d0, _ = Qm(x)
    Qm(x), Qm(x)
    with pytest.raises(RuntimeError, match="overwritten"):
        d0.sum().backward()
    with pytest.raises(RuntimeError, match="double backward"):
        Qm(x)[1].sum().backward(create_graph=True)


def test_entries_refuse_bad_arguments_before_any_launch():
    import gm_b200
    from gm_b200._lib import lib, _ptr, _stream
    eng = gan_engine("began", max_batch=64)
    x = torch.rand(8, 784, device="cuda")
    out = torch.empty(8, 784, device="cuda")
    _refused(lambda: eng.d_forward(0, x), "scalar-output discriminator")
    _refused(lambda: eng.d_backward(0, torch.ones(8, device="cuda"), True), "scalar-output discriminator")
    _refused(lambda: eng.ae_forward(2, x), "slot")
    _refused(lambda: eng.ae_backward(-1, out, False), "slot")
    _refused(lambda: eng.ae_forward(0, torch.rand(65, 784, device="cuda")), "batch")
    ns = gan_engine("ns", max_batch=64)
    _refused(lambda: ns.ae_forward(0, x), "GM_BEGAN")
    info = _info_engine(784, 400, 20, max_batch=64)
    codes = torch.empty(8, 20, device="cuda")
    _refused(lambda: info.q_forward(2, x), "slot")
    _refused(lambda: info.q_backward(0, torch.rand(65, 20, device="cuda"), False), "batch")
    split_began = gan_engine("began", max_batch=64, precision="split")
    _refused(lambda: split_began.ae_forward(0, x), "bf16 only")
    split_info = gm_b200.InfoGanEngine(784, 400, 20, max_batch=64, precision="split")
    _refused(lambda: split_info.q_forward(0, x), "bf16 only")
    # return codes straight from the C ABI: wrong engine kind, unbound Q, null pointers, nothing launched
    unbound = gm_b200.GanEngine(784, 400, 40, max_batch=64, variant="info")
    n0 = gm_b200.launch_count()
    s = _stream()
    assert lib().gm_gan_q_forward(eng.g, 0, _ptr(x), 8, _ptr(codes), s) == -4         # GM_ERR_UNSUPPORTED: not GM_INFO
    assert lib().gm_gan_q_backward(unbound.g, 0, 8, _ptr(codes), None, s) == -3      # GM_ERR_STATE: Q not bound
    assert lib().gm_gan_ae_forward(eng.g, 0, None, 8, _ptr(out), s) == -1
    assert lib().gm_gan_ae_forward(eng.g, 0, _ptr(x), 8, None, s) == -1
    assert lib().gm_gan_ae_backward(eng.g, 0, 8, None, None, s) == -1
    assert lib().gm_gan_q_forward(info.g, 0, None, 8, _ptr(codes), s) == -1
    assert lib().gm_gan_q_forward(info.g, 0, _ptr(x), 8, None, s) == -1
    assert lib().gm_gan_q_backward(info.g, 0, 8, None, None, s) == -1
    assert lib().gm_gan_q_forward(info.g, 0, _ptr(x), 0, _ptr(codes), s) == -1
    assert lib().gm_gan_ae_forward(None, 0, _ptr(x), 8, _ptr(out), s) == -1
    assert lib().gm_gan_num_q_slots(info.g) == 2 and lib().gm_gan_num_q_slots(eng.g) == 0
    assert gm_b200.launch_count() == n0
    # the G entries accept BEGAN engines
    img = eng.g_forward(torch.randn(8, 20, device="cuda"))
    assert torch.isfinite(eng.g_backward(torch.full_like(img, 1e-3))).all()


# ---------------------------------------------------------------- 7: launch ledger
def _check(fn):
    """gm_launch_count delta of fn() == this library's kernels in the CUDA trace (copies, memsets and torch's own at::
    kernels left out) == the launches gm_prof_report counts at level 2"""
    import gm_b200
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    gm_b200.prof_report()                     # drops records left by earlier calls
    gm_b200.prof_enable(2)
    try:
        n0 = gm_b200.launch_count()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        delta = gm_b200.launch_count() - n0
        report = sum(n for _, n, _ in gm_b200.prof_report())
    finally:
        gm_b200.prof_enable(0)
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset")) and "at::" not in e.name]
    assert delta == len(kernels) == report > 0, (delta, report, kernels)


def _ledger_of_the_new_entries():
    n = 32
    x = torch.rand(n, 784, device="cuda")
    eng = gan_engine("began", max_batch=64)
    _check(lambda: eng.ae_forward(1, x))
    dr = torch.full((n, 784), 1e-3, device="cuda")
    _check(lambda: eng.ae_backward(1, dr, True))
    _check(lambda: eng.ae_backward(1, dr, False))
    info = _info_engine(784, 400, 20, max_batch=64)
    info.q_forward(0, x)                              # the first call allocates the slot buffers
    _check(lambda: info.q_forward(1, x))
    dc = torch.full((n, 20), 1e-2, device="cuda")
    _check(lambda: info.q_backward(1, dc, True))
    _check(lambda: info.q_backward(1, dc, False))


def test_launch_ledger_of_the_new_entries():
    """for each of the four entries: gm_launch_count delta == library kernels in the CUDA trace == gm_prof_report total
    (the method of tests/test_launch_ledger_gpu.py).  The profiler sessions run in a child process, so this process's
    CUDA profiler state stays as the other tests find it."""
    import os
    import subprocess
    import sys
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(p for p in sys.path if p))
    r = subprocess.run([sys.executable, "-c", "import test_began_info_custom_gpu as t; t._ledger_of_the_new_entries()"],
                       cwd=os.path.dirname(os.path.abspath(__file__)), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
