"""User-written losses on the DCGAN conv path (README.md:31: "edit train_D and train_G"), on the GPU: the layout kernels
at the autograd boundary (gm_image_to_rows / gm_rows_to_image) bitwise against the torch expressions they replace, the
grad-mode forwards of model.G / model.D against the no-grad ones, their backward with generic upstreams against fp32
autograd at the bf16 storage points (oracle/dcgan_torch.py), the reference's NS loss and a hinge loss written in torch,
train() on an override against the reference loop in torch, and the errors for overwritten slots and double backward.
With GM_PARITY_DIR set, the measured errors are written to $GM_PARITY_DIR/parity_dcgan_custom.json."""
import ctypes as C

import numpy as np
import pytest
import torch

import dcgan_harness as H
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_custom")


# ---------------------------------------------------------------- the reference's NS loss (src/ns_gan.py:172-216), verbatim
def _ns_train_D(self, images):
    # Sample noise z, generate output G(z)
    noise = self.compute_noise(images.shape[0], self.model.z_dim)
    G_output = self.model.G(noise)

    # Classify the generated and real batch images
    DX_score = self.model.D(images) # D(x)
    DG_score = self.model.D(G_output) # D(G(z))

    # Compute vanilla (original paper) D loss
    D_loss = torch.sum(-torch.mean(torch.log(DX_score + 1e-8)
                        + torch.log(1 - DG_score + 1e-8)))

    return D_loss


def _ns_train_G(self, images):
    # Get noise (denoted z), classify it using G, then classify the output
    # of G using D.
    noise = self.compute_noise(images.shape[0], self.model.z_dim) # (z)
    G_output = self.model.G(noise) # G(z)
    DG_score = self.model.D(G_output) # D(G(z))

    # Compute the non-saturating loss for how D did versus the generations
    # of G using sigmoid cross entropy
    G_loss = -torch.mean(torch.log(DG_score + 1e-8))

    return G_loss


def _hinge_train_D(self, images):
    noise = self.compute_noise(images.shape[0], self.model.z_dim)
    return torch.mean(torch.relu(1 - self.model.D(images))) + torch.mean(torch.relu(1 + self.model.D(self.model.G(noise))))


def _hinge_train_G(self, images):
    noise = self.compute_noise(images.shape[0], self.model.z_dim)
    return -torch.mean(self.model.D(self.model.G(noise)))


def _recording(Trainer, train_D, train_G):
    """Trainer with the given steps, whose compute_noise / process_batch log what they hand out (replayed by the oracle)"""
    class Rec(Trainer):
        def compute_noise(self, batch_size, z_dim):
            z = self.noise_feed.pop(0).cuda() if self.noise_feed else super().compute_noise(batch_size, z_dim)
            self.noise_log.append(z.detach().cpu().clone())
            return z

        def process_batch(self, iterator):
            x = super().process_batch(iterator)
            self.batch_log.append(x.detach().cpu().clone())
            return x
    Rec.train_D, Rec.train_G = train_D, train_G
    return Rec


def _make(variant="ns", out_act="relu", hd=16, seed=11, wstd=0.05, Trainer=None, loader=None):
    """a conv drop-in model + trainer (Trainer, default the shipped one) with dcgan_harness.setup's weights (the same draws
    in the engine's layout, so the same operating point as the fused path's tests), and the oracle G / D with them.
    Returns (model, trainer, engine, G, D, the generator), the generator continuing setup's stream of draws."""
    import dc_gan
    import dc_w_gp_gan
    if variant == "ns":
        model = dc_gan.DCGAN(hidden_dim=hd, z_dim=100)
        Trainer = Trainer or dc_gan.DCGANTrainer
    else:
        model = dc_w_gp_gan.DCWGPGAN(hidden_dim=hd, z_dim=100, out_act=out_act)
        Trainer = Trainer or dc_w_gp_gan.DCWGPGANTrainer
    tr = Trainer(model, loader, loader, loader)
    tr.noise_log, tr.batch_log, tr.noise_feed = [], [], []
    eng = tr._engine_synced()
    g = torch.Generator().manual_seed(seed)
    for net in (eng.G, eng.D):
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.D.view("l5.weight")[1:].zero_()
    eng.G.refresh(); eng.D.refresh()
    sd = eng.torch_weights()
    with torch.no_grad():
        for k, p in model.named_parameters():
            p.copy_(sd[k])
    G = O.Generator(hd, 100)
    D = O.Discriminator(hd) if eng.d_bn else O.Critic(hd, 3, eng.d_out_act)
    O.load_from_engine_weights(G, D, eng.torch_weights())
    G.train(); D.train()
    G.q = staticmethod(O.bf16_points)
    if eng.d_bn:
        D.q = staticmethod(O.bf16_points)
    return model, tr, eng, G, D, g


def _oracle_scores(D, x):
    """D(x) of the oracle at the bf16 storage points (the critic takes its rounding per call)"""
    if isinstance(D, O.Critic):
        return D.out(D.trace(x, q=O.bf16_points)[0]).view(-1, 1)
    return D(x)


def _live_critic(model, tr, D, x):
    """flip the relu critic's last layer when fewer than half of x's rows are live (a dead row has zero gradient)"""
    if isinstance(D, O.Critic) and D.out_act == "relu" and int((D.trace(x, q=O.bf16_points)[0] > 0).sum()) < x.shape[0] // 2:
        with torch.no_grad():
            D.l5.weight.neg_()
            model.D.l5.weight.neg_()
        tr._dirty = True


# ---------------------------------------------------------------- 1. layout kernels
@pytest.mark.parametrize("n", [1, 7, 1024])
@pytest.mark.parametrize("ch", [1, 3])
def test_layout_kernels_are_bitwise_the_torch_expressions(ch, n):
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=16, channels=ch)
    g = torch.Generator(device="cuda").manual_seed(10 * n + ch)
    x = torch.randn(n, ch * 4096, device="cuda", generator=g)
    # round-to-nearest-even ties both ways, signed zeros, a subnormal
    x.view(-1)[:6] = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -0.0, 0.0, -(1 + 2 ** -8), 1e-40])
    nhwc = x.view(n, ch, 64, 64).permute(0, 2, 3, 1)
    rows = eng.stage_images(x)
    want = nhwc.to(torch.bfloat16).contiguous().view(n * 4096, ch)         # stage_images' previous torch expression
    assert torch.equal(rows.view(torch.int16), want.view(torch.int16))
    f = torch.rand(n * 4096, ch, device="cuda", generator=g).to(torch.bfloat16)
    up = eng.image_to_rows(x, f)
    gx, ff = nhwc.reshape(n * 4096, ch), f.float()
    assert torch.equal(up.view(torch.int16), (gx * ff * (1 - ff)).to(torch.bfloat16).view(torch.int16))
    back = eng.rows_to_image(rows, n)
    assert torch.equal(back, rows.view(n, 64, 64, ch).permute(0, 3, 1, 2).float().reshape(n, -1))
    # the wrapper takes [n, ch, 64, 64] and other dtypes through .float()
    u8 = torch.randint(0, 256, (n, ch, 64, 64), device="cuda", dtype=torch.uint8, generator=g)
    assert torch.equal(eng.stage_images(u8), u8.permute(0, 2, 3, 1).to(torch.bfloat16).reshape(n * 4096, ch))


def test_layout_kernels_refuse_bad_arguments_before_any_launch():
    from gm_b200 import _lib
    L, h, s, p = _lib.lib(), _lib.ctx(), _lib._stream(), _lib._ptr
    x = torch.zeros(2, 3 * 4096 + 4, device="cuda")
    rows = torch.zeros(2 * 4096 + 8, 3, device="cuda", dtype=torch.bfloat16)
    off = lambda t, b: C.c_void_p(t.data_ptr() + b)     # noqa: E731
    _lib.launch_count(reset=True)
    bad = [L.gm_image_to_rows(h, p(x), None, 0, 3, p(rows), s), L.gm_image_to_rows(h, p(x), None, -1, 3, p(rows), s),
           L.gm_image_to_rows(h, p(x), None, 2, 0, p(rows), s), L.gm_image_to_rows(h, p(x), None, 2, 5, p(rows), s),
           L.gm_image_to_rows(h, None, None, 2, 3, p(rows), s), L.gm_image_to_rows(h, p(x), None, 2, 3, None, s),
           L.gm_image_to_rows(h, off(x, 4), None, 2, 3, p(rows), s), L.gm_image_to_rows(h, p(x), off(rows, 2), 2, 3, p(rows), s),
           L.gm_image_to_rows(h, p(x), None, 2, 3, off(rows, 8), s), L.gm_image_to_rows(None, p(x), None, 2, 3, p(rows), s),
           L.gm_rows_to_image(h, p(rows), 0, 3, p(x), s), L.gm_rows_to_image(h, p(rows), 2, 5, p(x), s),
           L.gm_rows_to_image(h, None, 2, 3, p(x), s), L.gm_rows_to_image(h, p(rows), 2, 3, None, s),
           L.gm_rows_to_image(h, off(rows, 2), 2, 3, p(x), s), L.gm_rows_to_image(h, p(rows), 2, 3, off(x, 8), s)]
    assert bad == [-1] * len(bad)
    assert _lib.launch_count(reset=True) == 0
    assert L.gm_image_to_rows(h, p(x), None, 2, 3, p(rows), s) == 0 and L.gm_rows_to_image(h, p(rows), 2, 3, p(x), s) == 0
    assert _lib.launch_count(reset=True) == 2


# ---------------------------------------------------------------- 2. forward identity
@pytest.mark.parametrize("variant", ["ns", "wgp"])
def test_grad_mode_forwards_equal_the_no_grad_forwards(variant):
    model, tr, eng, _, _, g = _make(variant)
    n = 8
    x = torch.rand(n, 3 * 4096, generator=g).cuda()
    z = torch.randn(n, 100, generator=g).cuda()
    runs = list(eng.run_G.values()) + list(eng.run_D.values())
    start = [r.clone() for r in runs]
    outs = {}
    for grad in (False, True):
        for r, r0 in zip(runs, start):
            r.copy_(r0)
        with torch.set_grad_enabled(grad):
            gz, dx = model.G(z), model.D(x)
        assert gz.requires_grad == grad and dx.requires_grad == grad
        outs[grad] = (gz.detach(), dx.detach(), [r.clone() for r in runs])
    assert torch.equal(outs[False][0], outs[True][0]) and torch.equal(outs[False][1], outs[True][1])
    assert gz.shape == (n, 3 * 4096) and dx.shape == (n, 1)
    assert all(torch.equal(a, b) for a, b in zip(outs[False][2], outs[True][2]))
    assert all(not torch.equal(a, b) for a, b in zip(outs[True][2], start))           # every running statistic moved


# ---------------------------------------------------------------- 3. generic upstreams through the nodes
@pytest.mark.parametrize("variant,out_act", [("ns", None), ("wgp", "relu"), ("wgp", "none")], ids=["bn-sigmoid", "critic-relu", "critic-none"])
def test_backward_through_the_nodes_with_generic_upstreams(variant, out_act):
    """as tests/test_dcgan_gpu.py::test_backward_passes_with_generic_upstream_gradients, through model.D / model.G: every
    D .grad and x.grad, then every G .grad, against fp32 autograd of the oracle at the bf16 storage points"""
    model, tr, eng, G, D, g = _make(variant, out_act or "relu")
    n = 8
    x = torch.rand(n, 3 * 4096, generator=g)
    _live_critic(model, tr, D, x)
    up = torch.randn(n, 1, generator=g)
    xc = x.cuda().requires_grad_()
    model.D(xc).backward(up.cuda())
    xi = x.clone().requires_grad_()
    gr = torch.autograd.grad(_oracle_scores(D, xi), list(D.parameters()) + [xi], up)
    rep = {"D_" + k: nrel(p.grad, gref) for (k, p), gref in zip(model.D.named_parameters(), gr[:-1])}
    rep["D_dx"] = nrel(xc.grad, gr[-1])
    z = torch.randn(n, 100, generator=g)
    out = model.G(z.cuda())
    gup = torch.randn(n, 3 * 4096, generator=g)
    out.backward(gup.cuda())
    gg = torch.autograd.grad(G(z), list(G.parameters()), gup)
    rep.update({"G_" + k: nrel(p.grad, gref) for (k, p), gref in zip(model.G.named_parameters(), gg)})
    _REPORT.add("generic_upstream_" + (out_act or "bn"), rep)
    # Measured on H100 hosts: G 0.2 - 0.9 %; the critic 0.2 - 2.5 %, its image gradient 3.6 %; the batch-norm D 0.2 - 1.2 %
    # on one host and 0.3 - 3.6 % on another for the same inputs.  The oracle runs on the host CPU, whose conv rounding
    # moves a few (Leaky)ReLU inputs within 2^-9 of zero to the other slope at the bf16 points, and each such unit moves a
    # layer's gradient by a few per cent (DESIGN.md §6b).  The image gradient through sigma' (the dimg_mode defect this
    # guards against) is off by O(1)
    for k, v in rep.items():
        assert v < 5e-2, (k, v, rep)


# ---------------------------------------------------------------- 4. the reference's NS loss in torch
def test_reference_ns_loss_written_in_torch():
    """src/ns_gan.py:172-216 verbatim as the override: one D step, then one G step (no update in between) at hidden 16 and
    batch 8, (a) against the oracle, (b) against the fused d_grad / g_grad on the same weights, images and noise"""
    import dc_gan
    Tr = _recording(dc_gan.DCGANTrainer, _ns_train_D, _ns_train_G)
    model, tr, eng, G, D, _ = _make("ns", Trainer=Tr)
    n = 8
    g = torch.Generator().manual_seed(5)                 # the draws of test_dcgan_train_step_matches_the_torch_oracle
    imgs = torch.rand(n, 3 * 4096, generator=g)
    tr.noise_feed = [torch.randn(n, 100, generator=g), torch.randn(n, 100, generator=g)]
    Ld = tr.train_D(imgs.cuda())
    Ld.backward()
    gd = {k: p.grad.clone() for k, p in model.D.named_parameters()}
    for p in model.parameters():
        p.grad = None
    Lg = tr.train_G(imgs.cuda())
    Lg.backward()
    gg = {k: p.grad.clone() for k, p in model.G.named_parameters()}
    z1, z2 = tr.noise_log
    rep = {}
    # (a) the oracle
    Ld_ref = O.d_loss(G, D, imgs, z1)
    rep["a_D_loss"] = abs(Ld.item() - Ld_ref.item()) / abs(Ld_ref.item())
    for (k, _), gref in zip(D.named_parameters(), torch.autograd.grad(Ld_ref, list(D.parameters()))):
        rep["a_gradD_" + k] = nrel(gd[k], gref)
    Lg_ref = O.g_loss(G, D, z2)
    rep["a_G_loss"] = abs(Lg.item() - Lg_ref.item()) / abs(Lg_ref.item())
    for (k, _), gref in zip(G.named_parameters(), torch.autograd.grad(Lg_ref, list(G.parameters()))):
        rep["a_gradG_" + k] = nrel(gg[k], gref)
    # (b) the fused step
    Ld_f = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z1.cuda()).item()
    tg = eng.torch_grads()
    rep["b_D_loss"] = abs(Ld.item() - Ld_f) / abs(Ld_f)
    rep.update({"b_gradD_" + k: nrel(gd[k], tg["D." + k]) for k in gd})
    Lg_f = eng.g_grad(n, noise=z2.cuda()).item()
    tg = eng.torch_grads()
    rep["b_G_loss"] = abs(Lg.item() - Lg_f) / abs(Lg_f)
    rep.update({"b_gradG_" + k: nrel(gg[k], tg["G." + k]) for k in gg})
    _REPORT.add("ns_override_step", rep)
    assert rep["a_D_loss"] < 5e-3 and rep["a_G_loss"] < 1e-2, rep       # test_dcgan_train_step_matches_the_torch_oracle's bounds
    # The G gradients measured 6 - 7 % and up to 12.8 % of the oracle on different H100 hosts for the same inputs (the fused
    # step's are within 0.65 % of these, (b)): the oracle's CPU rounding at the bf16 points flips a few ReLU units, which
    # BatchNorm over 8 images amplifies through G's four layers (DESIGN.md §6b, the 20 % bound of the InfoGAN / VAE steps)
    for k, v in rep.items():
        if k.startswith("a_grad"):
            assert v < (0.12 if k.startswith("a_gradD") else 0.2), (k, v, rep)
    # (b): the losses come from the same logits through the same formulas (torch's log on the host side here, the loss kernel
    # there), and the D gradients differ only where sigma' is applied (torch on the n logits here, inside the loss kernel
    # there).  The G step also rounds dL/dG(z) (G's upstream from D's image gradient) to bf16 once before sigma' is applied,
    # where the fused step applies sigma' in the same col2im pass and rounds once
    assert rep["b_D_loss"] < 1e-5 and rep["b_G_loss"] < 1e-5, rep
    for k, v in rep.items():
        if k.startswith("b_gradD"):
            assert v < B_GRAD_D, (k, v, rep)
        if k.startswith("b_gradG"):
            assert v < B_GRAD_G, (k, v, rep)


# measured on an H100: the D gradients are equal (the override's sigma' on the n logits gives the same bf16 upstream as
# the loss kernel), the G gradients 0.35 - 0.65 % apart, the one bf16 rounding of dL/dG(z) before sigma' is applied
B_GRAD_D, B_GRAD_G = 1e-6, 2e-2


# ---------------------------------------------------------------- 5. a loss the fused path does not have
def test_hinge_loss_on_the_linear_critic():
    import dc_w_gp_gan
    Tr = _recording(dc_w_gp_gan.DCWGPGANTrainer, _hinge_train_D, _hinge_train_G)
    model, tr, eng, G, D, g = _make("wgp", "none", Trainer=Tr)
    n = 8
    imgs = torch.rand(n, 3 * 4096, generator=g)          # the draws of dcgan_harness.critic_setup("wgp", "none")
    z = torch.randn(n, 100, generator=g)
    tr.noise_feed = [z, z]
    Ld = tr.train_D(imgs.cuda())
    Ld.backward()
    gd = {k: p.grad.clone() for k, p in model.D.named_parameters()}
    for p in model.parameters():
        p.grad = None
    Lg = tr.train_G(imgs.cuda())
    Lg.backward()
    gg = {k: p.grad.clone() for k, p in model.G.named_parameters()}
    z1, z2 = tr.noise_log
    s = lambda x: _oracle_scores(D, x)                      # noqa: E731
    with torch.no_grad():
        fake_dev = model.G(z1.cuda()).cpu()                  # the images D received: G's forward is deterministic
    real, fake = torch.mean(torch.relu(1 - s(imgs))), torch.mean(torch.relu(1 + s(fake_dev)))
    Ld_ref = real + fake
    rep = {"D_loss": abs(Ld.item() - Ld_ref.item()) / abs(Ld_ref.item())}
    parts = [torch.autograd.grad(t, list(D.parameters()), retain_graph=True) for t in (real, fake)]
    for i, (k, _) in enumerate(D.named_parameters()):
        gref = parts[0][i] + parts[1][i]
        rep["gradD_" + k] = nrel(gd[k], gref)
        # as in test_dcgan_wgp_gpu's D step: the real and fake parts nearly cancel, so the bf16 rounding of each part shows
        # against the size of the parts, not of their sum
        scale = float(parts[0][i].norm() + parts[1][i].norm())
        rep["cancellation_" + k] = scale / float(gref.norm())
        rep["of_parts_" + k] = float((gd[k].cpu().double() - gref.double()).norm()) / scale
    sg = s(G(z2))
    Lg_ref = -torch.mean(sg)
    # -mean(D(G(z))) is a mean of signed scores: as test_dcgan_wgp_gpu holds the W part, against the size of its terms
    rep["G_loss"] = abs(Lg.item() - Lg_ref.item()) / float(sg.abs().mean())
    for (k, _), gref in zip(G.named_parameters(), torch.autograd.grad(Lg_ref, list(G.parameters()))):
        rep["gradG_" + k] = nrel(gg[k], gref)
    _REPORT.add("hinge_step", rep)
    # the D loss within tests/test_dcgan_wgp_gpu.py's bound; the G loss measured 3e-3 - 1.7e-2 of mean |D(G(z))| on three
    # H100 hosts for the same inputs: the oracle's G forward runs on the host CPU, and its rounding at the bf16 points moves
    # G(z), which the D-step comparison avoids by scoring the device's own G(z)
    assert rep["D_loss"] < 5e-3 and rep["G_loss"] < 5e-2, rep
    # the real and fake parts cancel to 1/3.5 - 1/8 of their size here (cancellation_*): the parts-relative error is the
    # precision measure, 0.1 - 1.1 % measured; the plain ratio reads 0.7 - 5.3 %
    for k, v in rep.items():
        if k.startswith("of_parts"):
            assert v < 3e-2, (k, v, rep)
        if k.startswith("gradD"):
            assert v < 6e-2, (k, v, rep)
        if k.startswith("gradG"):
            assert v < 0.12, (k, v, rep)


# ---------------------------------------------------------------- 6. train() honours the override
def test_train_runs_the_override_and_follows_the_reference_loop():
    import dc_gan
    from gm_b200 import _lib
    n, steps = 8, 3
    g0 = torch.Generator().manual_seed(2)
    data = torch.rand(steps * n, 3, 64, 64, generator=g0)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(data, torch.zeros(steps * n)), batch_size=n, shuffle=True)
    Tr = _recording(dc_gan.DCGANTrainer, _ns_train_D, _ns_train_G)
    model, tr, eng, G, D, g = _make("ns", Trainer=Tr, loader=loader)
    assert tr._has_custom_step()
    lr = 2e-4
    start = {k: v.detach().clone() for k, v in model.state_dict().items()}
    torch.manual_seed(7)
    _lib.launch_count(reset=True)
    tr.train(num_epochs=1, G_lr=lr, D_lr=lr)
    launches = _lib.launch_count(reset=True)
    assert launches > 50 * steps, launches                        # the forwards / backwards ran in libgm_b200.so
    assert len(tr.Dlosses) == steps and len(tr.Glosses) == steps
    # the reference loop in torch on the oracle model, with the same batches and noise
    Gopt, Dopt = torch.optim.Adam(G.parameters(), lr=lr), torch.optim.Adam(D.parameters(), lr=lr)
    rep, Dl, Gl = {}, [], []
    for i in range(steps):
        images, (z1, z2) = tr.batch_log[i], tr.noise_log[2 * i:2 * i + 2]
        Dopt.zero_grad()
        L = O.d_loss(G, D, images, z1)
        L.backward()
        Dopt.step()
        Dl.append(L.item())
        Gopt.zero_grad()
        L = O.g_loss(G, D, z2)
        L.backward()
        Gopt.step()
        Gl.append(L.item())
    rep["D_loss"] = [abs(a - b) / abs(b) for a, b in zip(tr.Dlosses, Dl)]
    rep["G_loss"] = [abs(a - b) / abs(b) for a, b in zip(tr.Glosses, Gl)]
    names = ["G." + k for k, _ in G.named_parameters()] + ["D." + k for k, _ in D.named_parameters()]
    ref = dict(zip(names, list(G.parameters()) + list(D.parameters())))
    sd = model.state_dict()
    flat = lambda d: torch.cat([d[k].detach().reshape(-1).cpu() for k in names])      # noqa: E731
    rep["params"] = nrel(flat(sd), flat(ref))
    rep["update"] = nrel(flat(sd) - flat(start), flat(ref) - flat(start))
    _REPORT.add("train_override", rep)
    # Measured on two H100 hosts: step-1 losses 1.1e-3 - 2.3e-3 (D) and 7.8e-4 - 5.8e-3 (G), within test 4's bounds; the
    # later steps up to 1.3e-2 (D) and 1.8e-2 (G); parameters 1.9e-3 - 2.0e-3.  Adam's first steps move a weight by about lr
    # times the sign of its gradient, so where a gradient is near zero the two loops move it opposite ways (the update
    # vectors are 0.27 - 0.29 apart) and steps 2 and 3 evaluate the losses at slightly different parameters
    assert rep["D_loss"][0] < 5e-3 and rep["G_loss"][0] < 1e-2, rep
    assert max(rep["D_loss"]) < TRAIN_LOSS_D and max(rep["G_loss"]) < TRAIN_LOSS_G, rep
    assert rep["params"] < TRAIN_PARAMS and rep["update"] < TRAIN_UPDATE, rep
    assert all(np.isfinite(tr.Dlosses)) and all(np.isfinite(tr.Glosses))
    # the engine's running statistics came back to the modules
    assert torch.equal(model.D.bn2.running_mean.cpu(), eng.run_D[1][0].cpu())
    assert torch.equal(model.G.bn1.running_var.cpu(), eng.run_G[0][1].cpu())


TRAIN_LOSS_D, TRAIN_LOSS_G, TRAIN_PARAMS, TRAIN_UPDATE = 2.5e-2, 4e-2, 5e-3, 0.5


# ---------------------------------------------------------------- 7. errors, not corruption
def test_overwritten_slots_and_double_backward_raise():
    model, tr, eng, _, _, g = _make("ns")
    n = 4
    x = torch.rand(n, 3 * 4096, generator=g).cuda()
    z = torch.randn(n, 100, generator=g).cuda()
    first = model.D(x)
    live = [model.D(x) for _ in range(3)]
    live[-1].sum().backward()                                   # four live D calls fit
    model.D(x)                                                  # a fifth takes the first call's slot
    with pytest.raises(RuntimeError, match="overwritten"):
        first.sum().backward()
    first_g = model.G(z)
    model.G(z)
    model.G(z)
    with pytest.raises(RuntimeError, match="overwritten"):
        first_g.sum().backward()
    xg = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(model.D(xg).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(model.G(z).sum(), list(model.G.parameters()), create_graph=True)
