"""The MLP engines (GanEngine, InfoGanEngine, VaeEngine) against the float64 numpy oracle at every width class the
engines accept, not only the reference's 784 / 400 / 20.

Much of the engines' layout and routing is derived from (image X, hidden H, z Z): the padded row lengths
XP = rup(X+1, 16), HP = rup(H+1, 16), ZP = rup(Z+1, 64) and the ones column each weight-gradient GEMM takes its bias
gradient from; the 2 cdiv(H, 208) row-dot slots of D's logit (2 cdiv(X, 208) for the penalty's ||V||^2); the GEMM
route of each product (the 64-wide K-major kernel for N <= 64, the 208-wide clustered or 256-wide M-major tile for the
weight gradients); G's first layer at K = rup(Z, 16); the multi-block loss passes once a batch has more than 256 rows.

Geometries (X, H, Z): (16, 16, 1) puts every product on the 64-wide kernels with 2 slots; (64, 64, 63) is the upper
edge of those kernels with the ones column the last one of ZP = 64; (208, 208, 64) is one full 208 tile and ZP = 128;
(3072, 224, 100) gives 48 k-blocks in D's first layer, a second 208 tile holding 16 columns and 30 penalty slots;
(1024, 432, 447) is the largest accepted H and Z (HP = ZP = 448, 6 slots, G's first layer at 7 k-blocks); (784, 400, 20)
is the reference's geometry, kept as the control.  One engine per (geometry, variant, precision), max_batch 320, runs
batches 1, 65 and 300 in turn: 300 gives the D step 600 logit rows, 3 blocks of the loss passes.

Tolerances and why:
  - Losses and D scores: 1e-3 relative (WGAN-GP's ReLU scores 3e-3: its raw outputs are O(0.05), so the absolute error
    of the sigmoid critics' O(0.5) outputs reads ~10x larger), gradients: 1e-3 norm-relative.  These are the bounds of
    test_gan_step_gpu.py (bf16 operands against the oracle evaluated at the same bf16 storage points,
    q = R.bf16_points) and of test_split_precision_gpu.py (split operands against the exact oracle).  Loss errors are
    measured against max(|loss|, 1e-3): WGAN-type losses are differences of O(1) means and can be ~0.
  - ReLU kinks: hidden units with |pre-activation| < TOL_A (2e-5, ~10 sigma of the fp32 / split-operand rounding of
    a 3072-term dot product) take the device's side (mlp_harness.DeviceReluSides, and VaeReluSides for the VAE's
    encoder and decoder layers).  Their count is reported and capped per step at 8 + 2e-4 of the hidden units the
    step evaluates (measured: at most ~5e-5 of them).  WGAN is capped at 15 %: its clamp puts every weight and bias
    at +-0.01 and the images are binary, so pre-activations lie on a lattice of multiples of 0.01 and a share of
    them cancel to zero exactly up to rounding (measured up to 8 % of a step's units at 16-wide layers).
  - bf16 mode, G step: G's hidden-layer gradient DHg = bf16((DA2 W2) * relu'(h)) is a sum over X products that can
    cancel, so its fp32 accumulation error is bounded by the sum of the magnitudes of its terms, not by its value:
    a few of its bf16 roundings land one or more ulps from the float64 model's (measured 1.008e-3 on G's first-layer
    gradient at batch 1, X = 3072).  The test checks every stored DHg element against the float64 product of the
    device's own DA2 rows: |DHg - e| <= 2^-8 |e| + (1 + 2^-8) 2 X u sum_k |DA2_k W2_kj| (bf16 products are exact
    in fp32, each of the X accumulating additions rounds by at most 2u whatever the rounding mode, the bf16 store by
    half an ulp, at most 2^-8 of the value with bf16's 8-bit significand), then evaluates G's first-layer gradients at the stored DHg.  DA2 itself is checked through
    G.generate's gradient, which is formed from it.
  - bf16 mode: G's output is taken as the device stored it, after checking every element is within one bf16 ulp of
    the model's (mlp_harness.DeviceReluSides, fake_rows): a one-ulp rounding difference of a fake element moves D's
    pre-activation on that row beyond TOL_A.
  - WGAN's db2 is a difference of two near-equal sums: its error is measured against the sum of the magnitudes of
    its terms.
  - BEGAN in bf16: 2e-2 on the gradients against the bf16-point oracle (test_gan_step_gpu.py's bound): sign(r - x)
    is discontinuous and flips where |r - x| is below the bf16 resolution of r.
  - Adam, elementwise, from the engine's own fp32 gradient and moments (u = 2^-24): every fp32 operation of
    adam_kernel is correctly rounded.  m = b1 m + (1-b1) g carries at most 3 roundings of its terms,
    |dm| <= 3u S with S = b1|m| + (1-b1)|g|; likewise |dv| <= 3u v (all terms positive).  The step
    (lr / bc1) m / (sqrt(v) / sqrt(bc2) + eps) then adds at most 9 relative roundings on top of dm (sqrt, two
    divisions, a product, the eps sum, the bias corrections), so |d step| <= 12u (lr / bc1) S / denom, and the
    subtraction rounds to half an ulp of the result: |dp| <= u |p| + 16u (lr / bc1) S / denom (12 -> 16 for slack).
    The WGAN clamp is 1-Lipschitz and exact, so the bound carries through it.
  - Padding: the ones column must hold exactly 1.0 and every column beyond it exactly 0 (the GEMMs that read these
    rows take the bias gradient from that column and rely on the zeros).

Measured worst error-to-bound ratios go to $GM_PARITY_DIR/parity_mlp_geometry.json."""
import numpy as np
import pytest
import torch

from dcgan_harness import Report
from inputs import gm_init_weights, params_dict
from mlp_harness import DeviceReluSides, VaeReluSides, aux_from, gan_engine, gan_shapes, nrel
from oracle import ref_math as R

pytestmark = pytest.mark.gpu

ROW_VARIANTS = ["ns", "mm", "ls", "w", "ra", "fisher", "f_total_variation", "f_forward_kl", "f_reverse_kl",
                "f_pearson", "f_hellinger", "f_jensen_shannon"]
GP_VARIANTS = ["wgp", "dra"]
CORE = ["ns", "ls", "ra", "fisher", "wgp", "dra"]
SMALL, EDGE64, TILE208, WIDE, LARGEST, CONTROL = (16, 16, 1), (64, 64, 63), (208, 208, 64), (3072, 224, 100), \
    (1024, 432, 447), (784, 400, 20)
GEOMS = [SMALL, EDGE64, TILE208, WIDE, LARGEST, CONTROL]
BATCHES = (1, 65, 300)
MAX_BATCH = 320
PRECISIONS = ("bf16", "split")
TOL, TOL_WGP_SCORE, TOL_BEGAN_BF16 = 1e-3, 3e-3, 2e-2
U = 2.0 ** -24
D_NAMES = ["D.linear.weight", "D.linear.bias", "D.discriminate.weight", "D.discriminate.bias"]
G_NAMES = ["G.linear.weight", "G.linear.bias", "G.generate.weight", "G.generate.bias"]
Q_NAMES = ["Q.linear.weight", "Q.linear.bias", "Q.inference.weight", "Q.inference.bias"]
REPORT = Report("mlp_geometry")


def _gid(g):
    return "%dx%dx%d" % g


def _cases():
    out = []
    for geom in GEOMS:
        for variant in (ROW_VARIANTS + GP_VARIANTS if geom in (SMALL, LARGEST) else CORE):
            for prec in PRECISIONS:
                out.append(pytest.param(geom, variant, prec, id="%s-%s-%s" % (_gid(geom), variant, prec)))
    return out


class Checks:
    """error / bound ratios of one case; fails at the end with all of them in the message"""

    def __init__(self):
        self.ratios, self.notes = {}, {}

    def add(self, key, err, bound):
        self.ratios[key] = max(self.ratios.get(key, 0.0), float(err) / bound)

    def rel(self, key, got, ref, bound=TOL, floor=1e-3):
        self.add(key, abs(float(got) - float(ref)) / max(abs(float(ref)), floor), bound)

    def tensors(self, prefix, got, ref, names, bound=TOL):
        for nme, g in zip(names, got):
            self.add(prefix + nme, nrel(g, ref[nme]), bound)

    def finish(self, key):
        worst = max(self.ratios, key=self.ratios.get)
        REPORT.add(key, dict(worst=self.ratios[worst], worst_of=worst, **self.notes,
                             ratios={k: round(v, 4) for k, v in self.ratios.items()}))
        bad = {k: v for k, v in self.ratios.items() if not v < 1.0}
        assert not bad, (key, bad, self.notes)


def _params(eng, net, names):
    return {n: v.detach().cpu().numpy().astype(np.float64) for n, v in zip(names, eng.views(net))}


def _snapshot(*tensors):
    return [t.detach().cpu().numpy().astype(np.float64) for t in tensors]


def _check_adam(ck, key, before, after, lr, step, clamp=0.0):
    """after = (p, m, v) of the engine; before = (p, g, m, v): a float64 Adam on the engine's own inputs"""
    p0, g, m0, v0 = before
    p1, m1, v1 = after
    b1, b2, eps = float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8))
    lr = float(np.float32(lr))
    bc1 = float(np.float32(1.0 - b1 ** step))            # the host's bias corrections, from the fp32 betas
    bc2s = float(np.float32(np.sqrt(1.0 - b2 ** step)))
    S = b1 * np.abs(m0) + (1 - b1) * np.abs(g)
    m = b1 * m0 + (1 - b1) * g
    v = b2 * v0 + (1 - b2) * g * g
    den = np.sqrt(v) / bc2s + eps
    p = p0 - (lr / bc1) * (m / den)
    if clamp:
        p = np.clip(p, -float(np.float32(clamp)), float(np.float32(clamp)))
    tiny = 1e-45
    ck.add(key + "_m", np.max(np.abs(m1 - m) / (3 * U * S + tiny)), 1.0)
    ck.add(key + "_v", np.max(np.abs(v1 - v) / (3 * U * v + tiny)), 1.0)
    ck.add(key + "_p", np.max(np.abs(p1 - p) / (U * np.abs(p) + 16 * U * (lr / bc1) * S / den + tiny)), 1.0)


def _check_padding(ck, eng, which, row0, rows, col, ld):
    v = eng.debug_read(which, row0, rows, ld).cpu().numpy()
    bad = int(np.count_nonzero(v[:, col] != 1.0)) + int(np.count_nonzero(v[:, col + 1:]))
    ck.add("pad_%s_%d" % (which, row0), bad, 0.5)


def _rup(a, m):
    return (a + m - 1) // m * m


def _gan_padding(ck, eng, X, H, Z, b, d_step):
    """the ones column and zero tail of the staged noise, G's hidden rows and the real / fake image rows"""
    _check_padding(ck, eng, "Zb", 0, b, Z, _rup(Z + 1, 64))
    _check_padding(ck, eng, "Hg", 0, b, H, _rup(H + 1, 16))
    _check_padding(ck, eng, "Xall", b, b, X, _rup(X + 1, 16))
    if d_step:
        _check_padding(ck, eng, "Xall", 0, b, X, _rup(X + 1, 16))


def _draws(rng, variant, b, X, Z):
    x = (rng.random((b, X)) < 0.3).astype(np.float32)
    z1 = rng.standard_normal((b, Z)).astype(np.float32)
    z2 = rng.standard_normal((b, Z)).astype(np.float32)
    extra = []
    if variant == "wgp":
        extra = [rng.random((b, 1)).astype(np.float32)]
    elif variant == "dra":
        extra = [rng.random((b, 1)).astype(np.float32), rng.random((b, X)).astype(np.float32)]
    return x, z1, z2, extra


def _d_step(ck, eng, tag, variant, prec, x, z1, extra, P, q):
    """one D step against the oracle at P -> (oracle's Fisher state or None, relu boundary count)"""
    b = x.shape[0]
    H = eng.hidden_dim
    aux_o, aux_d = aux_from(iter(extra), variant)
    st = None
    if variant == "fisher":
        lam, rho = eng.fisher_state()
        st = dict(LAMBDA=np.float64(lam), RHO=np.float64(rho))
    Ld = eng.d_grad(torch.from_numpy(x).cuda(), noise=torch.from_numpy(z1).cuda(), aux=aux_d).item()
    sc = eng.scores(2 * b).cpu().numpy()
    gD = [t.cpu().numpy() for t in eng.views(1, eng.grads[1])]
    pre = None
    if variant == "wgp" and prec == "bf16":
        # the x_hat rows are never formed: the bf16-point model takes a_hat from the STORED pre-activations of the real /
        # fake rows (test_gan_step_gpu.py)
        a = eng.debug_read("Aall", 0, 2 * b, H).cpu().numpy().astype(np.float64)
        pre = (a[:b], a[b:])
    regions = [("Aall", 0, True), ("Aall", 1, True), ("DHall", 2)] if variant == "wgp" else [0, 1, 2]
    with DeviceReluSides(eng, d_regions=regions, g_hidden=False, fake_rows=_fake_rows(prec)) as sides:
        Lo, go, info = R.gan_d_step(P, variant, x.astype(np.float64), z1.astype(np.float64), aux_o, st, q=q, pre_points=pre)
    ck.rel(tag + "D_loss", Ld, Lo)
    tol_s = TOL_WGP_SCORE if variant == "wgp" else TOL
    ck.add(tag + "DX_score", nrel(sc[:b], info["dx"]), tol_s)
    ck.add(tag + "DG_score", nrel(sc[b:], info["dg"]), tol_s)
    ck.tensors(tag + "grad_", gD[:3], go, D_NAMES[:3])
    db2 = go["D.discriminate.bias"][0]
    scale = abs(db2)
    if variant == "w":
        # WGAN's db2 = (sum over fake rows of d(1-d) - the same over real rows) / B: two near-equal sums once the clamp
        # makes D nearly constant, so its error is bounded relative to the sum of the magnitudes of its terms
        scale = max(scale, float(np.sum(info["dx"] * (1 - info["dx"])) + np.sum(info["dg"] * (1 - info["dg"]))) / b)
    ck.add(tag + "grad_D.discriminate.bias", abs(float(gD[3][0]) - db2) / max(scale, 1e-30), TOL)
    if variant == "fisher":
        # lambda += rho * dL/dlambda, applied on the device by the loss pass's last block
        lam1, rho = eng.fisher_state()
        ref = st["LAMBDA"] + st["RHO"] * st["dLAMBDA"]
        ck.add(tag + "fisher_lambda", abs(lam1 - ref), TOL * rho * max(abs(st["dLAMBDA"]), 1.0) + 4 * U * abs(ref))
    return sides.count, sides.fake_flips


def _relu_cap(variant, units):
    """most near-kink units one step may hand to the device (see the module docstring)"""
    return 0.15 * units if variant == "w" else 8 + 2e-4 * units


class StoredDhg:
    """bf16 mode, G step: G's first-layer gradients from the device's stored dL/dh of G (DHg), after checking DHg
    elementwise against the float64 product of the device's own DA2 rows with the bf16 W2 (see the module docstring)."""

    def __init__(self, eng, on):
        self.eng, self.on, self.ratio = eng, on, 0.0

    def __enter__(self):
        self._gb = R.g_backward
        if not self.on:
            return self

        def g_backward(P, fw, dout, pre="G.", q=R._exact):
            g = self._gb(P, fw, dout, pre=pre, q=q)
            n, X = fw["out"].shape
            H = fw["h"].shape[1]
            da2 = self.eng.debug_read("DA2", 0, n, X).cpu().numpy().astype(np.float64)
            W2 = q("W", P[pre + "generate.weight"])
            mask = fw["h"] > 0
            exact = (da2 @ W2) * mask
            terms = (np.abs(da2) @ np.abs(W2)) * mask
            dev = self.eng.debug_read("DHg", 0, n, H).cpu().numpy().astype(np.float64)
            bound = 2.0 ** -8 * np.abs(exact) + (1 + 2.0 ** -8) * 2 * X * U * terms
            self.ratio = max(self.ratio, float(np.max(np.abs(dev - exact) / (bound + 1e-45))))
            g[pre + "linear.weight"] = dev.T @ fw["z"]
            g[pre + "linear.bias"] = dev.sum(0)
            return g
        R.g_backward = g_backward
        return self

    def __exit__(self, *exc):
        R.g_backward = self._gb
        return False


def _fake_rows(prec):
    """bf16 mode: the oracle takes G's output as stored (mlp_harness.DeviceReluSides)"""
    return 1 if prec == "bf16" else None


@pytest.mark.parametrize("geom,variant,prec", _cases())
def test_gan_steps_adam_and_padding(geom, variant, prec):
    import gm_b200
    X, H, Z = geom
    eng = gan_engine(variant, X, H, Z, max_batch=MAX_BATCH, precision=prec)
    q = R.bf16_points if prec == "bf16" else R._exact
    names = [n for n, _ in gan_shapes(X, H, Z)]
    gn = [n + s for n in names[:2] for s in (".weight", ".bias")]
    dn = [n + s for n in names[2:] for s in (".weight", ".bias")]
    assert gn == G_NAMES and dn == D_NAMES
    lr, clamp = 1e-3, (0.01 if variant == "w" else 0.0)
    hpD, hpG = gm_b200.AdamHP.make(lr, clamp=clamp), gm_b200.AdamHP.make(lr)
    if variant == "fisher":
        eng.fisher_state(0.5, 0.1)   # a nonzero lambda and rho: the moments reach the gradients and the lambda update
    rng = np.random.default_rng([X, H, Z, sum(map(ord, variant))])
    ck = Checks()
    relu, evaluated, flips = 0, 0, 0
    for step, b in enumerate(BATCHES, start=1):
        x, z1, z2, extra = _draws(rng, variant, b, X, Z)
        tag = "b%d_" % b
        P = {**_params(eng, 0, G_NAMES), **_params(eng, 1, D_NAMES)}
        n, f = _d_step(ck, eng, tag, variant, prec, x, z1, extra, P, q)
        relu, flips = relu + n, flips + f
        evaluated += (3 if variant in GP_VARIANTS else 2) * b * H
        ck.add("relu_units_at_boundary", n, _relu_cap(variant, (3 if variant in GP_VARIANTS else 2) * b * H))
        _gan_padding(ck, eng, X, H, Z, b, True)
        before = _snapshot(eng.params[1], eng.grads[1], eng.exp_avg[1], eng.exp_avg_sq[1])
        eng.apply(1, hpD)
        _check_adam(ck, tag + "adam_D", before, _snapshot(eng.params[1], eng.exp_avg[1], eng.exp_avg_sq[1]),
                    lr, step, clamp)
        # the G step runs D at its updated parameters: D's bf16 operand copies come from the Adam kernel's shadow writes
        P = {**_params(eng, 0, G_NAMES), **_params(eng, 1, D_NAMES)}
        Lg = eng.g_grad(b, noise=torch.from_numpy(z2).cuda()).item()
        scg = eng.scores(2 * b).cpu().numpy()[b:]
        gG = [t.cpu().numpy() for t in eng.views(0, eng.grads[0])]
        with DeviceReluSides(eng, d_regions=[1], fake_rows=_fake_rows(prec)) as sides, StoredDhg(eng, prec == "bf16") as dhg:
            Lgo, ggo, ginfo = R.gan_g_step(P, variant, z2.astype(np.float64), q=q)
        relu, flips = relu + sides.count, flips + sides.fake_flips
        ck.add("relu_units_at_boundary", sides.count, _relu_cap(variant, 2 * b * H))
        if dhg.on:
            ck.add(tag + "G_dhg_stored", dhg.ratio, 1.0)
        evaluated += 2 * b * H
        ck.rel(tag + "G_loss", Lg, Lgo)
        ck.add(tag + "G_score", nrel(scg, ginfo["dg"]), TOL_WGP_SCORE if variant == "wgp" else TOL)
        ck.tensors(tag + "grad_", gG, ggo, G_NAMES)
        _gan_padding(ck, eng, X, H, Z, b, False)
        before = _snapshot(eng.params[0], eng.grads[0], eng.exp_avg[0], eng.exp_avg_sq[0])
        eng.apply(0, hpG)
        _check_adam(ck, tag + "adam_G", before, _snapshot(eng.params[0], eng.exp_avg[0], eng.exp_avg_sq[0]),
                    lr, step)
    # one more D step at the parameters the last two Adam steps produced (G's and D's bf16 copies from adam_segs)
    x, z1, _, extra = _draws(rng, variant, 65, X, Z)
    P = {**_params(eng, 0, G_NAMES), **_params(eng, 1, D_NAMES)}
    n, f = _d_step(ck, eng, "final_", variant, prec, x, z1, extra, P, q)
    relu, flips = relu + n, flips + f
    evaluated += (3 if variant in GP_VARIANTS else 2) * 65 * H
    ck.add("relu_units_at_boundary", n, _relu_cap(variant, (3 if variant in GP_VARIANTS else 2) * 65 * H))
    ck.notes.update(relu_units_at_boundary=relu, hidden_units_evaluated=evaluated, fake_elements_one_ulp_off=flips)
    ck.finish("gan_%s_%s_%s" % (_gid(geom), variant, prec))


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("geom", [SMALL, (1024, 432, 427)], ids=_gid)
def test_infogan_q_step(geom, prec):
    """InfoGAN's mutual-information step: the MI loss and the G and Q gradients.  The generator input is z + 20 codes
    wide, so z = 427 is the largest accepted."""
    import gm_b200
    X, H, z = geom
    Z = z + 20
    shapes = [("G.linear", (H, Z)), ("G.generate", (X, H)), ("D.linear", (H, X)), ("D.discriminator", (1, H)),
              ("Q.linear", (H, X)), ("Q.inference", (20, H))]
    W = gm_init_weights(shapes, 1234)
    eng = gm_b200.InfoGanEngine(X, H, z, 10, 10, max_batch=MAX_BATCH, precision=prec)
    eng.load(0, [W["G.linear"][0], W["G.linear"][1], W["G.generate"][0], W["G.generate"][1]])
    eng.load(1, [W["D.linear"][0], W["D.linear"][1], W["D.discriminator"][0], W["D.discriminator"][1]])
    eng.load_q([W["Q.linear"][0], W["Q.linear"][1], W["Q.inference"][0], W["Q.inference"][1]])
    P = {k.replace("D.discriminator", "D.discriminate"): v for k, v in params_dict(W, np.float64).items()}
    q = R.bf16_points if prec == "bf16" else R._exact
    rng = np.random.default_rng([X, H, z, 7])
    ck = Checks()
    relu = 0
    for b in BATCHES:
        noise = np.zeros((b, Z), np.float32)
        noise[:, :z] = rng.standard_normal((b, z))
        noise[np.arange(b), z + rng.integers(0, 10, b)] = 1.0
        noise[:, z + 10:] = rng.uniform(-1, 1, (b, 10))
        L = eng.q_grad(b, torch.from_numpy(noise).cuda()).item()
        gG = [t.cpu().numpy() for t in eng.views(0, eng.grads[0])]
        gQ = [t.cpu().numpy() for t in eng.q_views(eng.q_grads)]
        with DeviceReluSides(eng, d_regions=[0], fake_rows=_fake_rows(prec)) as sides:
            Lo, go = R.info_q_step(P, noise.astype(np.float64), z_dim=z, q=q)
        relu += sides.count
        tag = "b%d_" % b
        ck.rel(tag + "MI_loss", L, Lo)
        ck.tensors(tag + "grad_", gG, go, G_NAMES)
        ck.tensors(tag + "grad_", gQ, go, Q_NAMES)
    ck.notes.update(relu_units_at_boundary=relu)
    ck.finish("info_%s_%s" % (_gid(geom), prec))


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("geom", [SMALL, WIDE, LARGEST], ids=_gid)
def test_began_steps_and_k_control(geom, prec):
    """BEGAN: the D step's loss, its DX / DG statistics and gradients, the G step, and the K controller fed by DX / DG."""
    X, H, Z = geom
    eng = gan_engine("began", X, H, Z, max_batch=MAX_BATCH, precision=prec)
    q = R.bf16_points if prec == "bf16" else R._exact
    tol_g = TOL_BEGAN_BF16 if prec == "bf16" else TOL
    enc = ["D.encoder.weight", "D.encoder.bias", "D.decoder.weight", "D.decoder.bias"]
    rng = np.random.default_rng([X, H, Z, 11])
    ck = Checks()
    K, gamma, lam = 0.3, 0.5, 0.05
    for b in BATCHES:
        x, z1, z2, _ = _draws(rng, "began", b, X, Z)
        tag = "b%d_" % b
        P = {**_params(eng, 0, G_NAMES), **_params(eng, 1, enc)}
        eng.began_init(K, b)
        Ld = eng.d_grad(torch.from_numpy(x).cuda(), noise=torch.from_numpy(z1).cuda()).item()
        st = eng.began_state()
        Lo, go, DX, DG = R.began_d_step(P, x.astype(np.float64), z1.astype(np.float64), K, q=q)
        ck.rel(tag + "D_loss", Ld, Lo)
        ck.rel(tag + "DX", st[3], DX)
        ck.rel(tag + "DG", st[4], DG)
        ck.tensors(tag + "grad_", [t.cpu().numpy() for t in eng.views(1, eng.grads[1])], go, enc, tol_g)
        Lg = eng.g_grad(b, noise=torch.from_numpy(z2).cuda()).item()
        Lgo, ggo = R.began_g_step(P, z2.astype(np.float64), q=q)
        ck.rel(tag + "G_loss", Lg, Lgo)
        ck.tensors(tag + "grad_", [t.cpu().numpy() for t in eng.views(0, eng.grads[0])], ggo, G_NAMES, tol_g)
        eng.began_control(gamma, lam, 5)
        K_ref = min(max(0.0, K + lam * (gamma * DX - DG)), 1.0)
        K = eng.began_state()[0]
        # K moves by lam (gamma DX - DG): the 1e-3 relative bound on DX and DG carries over, plus fp32 rounding of K
        ck.add(tag + "K", abs(K - K_ref), TOL * lam * (gamma * abs(DX) + abs(DG)) + 4 * U)
    ck.finish("began_%s_%s" % (_gid(geom), prec))


VAE_GEOMS = [(16, 16, 2), (64, 64, 32), (3072, 224, 8), (1024, 432, 20)]   # odd z is refused (decoder bias alignment)


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("geom", VAE_GEOMS, ids=_gid)
def test_vae_steps_and_adam(geom, prec):
    """VaeEngine: recon, KL and all ten gradient tensors at batches 1, 65 and 300, with Adam steps in between (each later
    batch runs at the parameters and bf16 operand copies the Adam kernel wrote).  z = 32 fills the 64-wide head."""
    import gm_b200
    X, H, Z = geom
    eng = gm_b200.VaeEngine(X, H, Z, max_batch=MAX_BATCH, precision=prec)
    shapes = [("encoder.linear", (H, X)), ("encoder.mu", (Z, H)), ("encoder.log_var", (Z, H)),
              ("decoder.linear", (H, Z)), ("decoder.recon", (X, H))]
    W = gm_init_weights(shapes, 4321)
    eng.load({k + s: v for k, (w, bb) in W.items() for s, v in ((".weight", w), (".bias", bb))})
    q = R.bf16_points if prec == "bf16" else R._exact
    lr = 1e-3
    hp = gm_b200.AdamHP.make(lr)
    rng = np.random.default_rng([X, H, Z, 13])
    ck = Checks()
    relu = 0
    for step, b in enumerate(BATCHES, start=1):
        x = (rng.random((b, X)) < 0.3).astype(np.float32)
        eps = rng.standard_normal((b, Z)).astype(np.float32)
        P = {k: v.cpu().numpy().astype(np.float64) for k, v in eng.views().items()}
        ls = eng.grad(torch.from_numpy(x).cuda(), eps=torch.from_numpy(eps).cuda()).cpu().numpy()
        gv = {k: v.cpu().numpy() for k, v in eng.views(eng.grads).items()}
        sides = VaeReluSides(eng)
        recon, kl, go, _ = R.vae_step(P, x.astype(np.float64), eps.astype(np.float64), q=q, relu=sides)
        tag = "b%d_" % b
        relu += sides.count
        ck.add("relu_units_at_boundary", sides.count, _relu_cap("vae", 2 * b * H))
        ck.rel(tag + "recon", ls[0], recon)
        ck.rel(tag + "kl", ls[1], kl)
        ck.tensors(tag + "grad_", [gv[k] for k in eng.NAMES], go, eng.NAMES)
        before = _snapshot(eng.params, eng.grads, eng.exp_avg, eng.exp_avg_sq)
        eng.apply(hp)
        _check_adam(ck, tag + "adam", before, _snapshot(eng.params, eng.exp_avg, eng.exp_avg_sq), lr, step)
    ck.notes.update(relu_units_at_boundary=relu)
    ck.finish("vae_%s_%s" % (_gid(geom), prec))


# ---------------------------------------------------------------- refusals


@pytest.mark.parametrize("kind,args", [
    ("gan", (784, 448, 20)), ("gan", (784, 400, 448)), ("gan", (792, 400, 20)), ("gan", (784, 0, 20)),
    ("info", (784, 400, 428)), ("vae", (784, 400, 33)), ("vae", (16, 16, 1)), ("vae", (784, 400, 19))],
    ids=["gan_H448", "gan_Z448", "gan_X792", "gan_H0", "info_z428", "vae_z33", "vae_z1", "vae_z19"])
def test_unsupported_widths_are_refused_without_launching(kind, args):
    import gm_b200
    n0 = gm_b200.launch_count()
    with pytest.raises(gm_b200.GmError):
        if kind == "gan":
            gm_b200.GanEngine(*args, max_batch=8)
        elif kind == "info":
            gm_b200.InfoGanEngine(args[0], args[1], args[2], 10, 10, max_batch=8)
        else:
            gm_b200.VaeEngine(*args, max_batch=8)
    assert gm_b200.launch_count() == n0


@pytest.mark.parametrize("variant", ["ns", "dra"])
def test_debug_read_refuses_rows_past_the_buffer(variant):
    """gm_gan_debug_read bounds row0 + rows by the buffer's row count: max_batch for Zb / Hg / DA2 / DHg, nreg x
    max_batch for Xall / Aall / DHall (nreg = 2, or 4 for DRAGAN's x_hat and penalty rows)"""
    import gm_b200
    Bm = 8
    eng = gan_engine(variant, 16, 16, 1, max_batch=Bm)
    nreg = 4 if variant == "dra" else 2
    for which in ("Zb", "Hg", "DA2", "DHg", "Xall", "Aall", "DHall"):
        n = Bm * (nreg if which in ("Xall", "Aall", "DHall") else 1)
        assert eng.debug_read(which, 0, n, 16).shape == (n, 16)
        assert eng.debug_read(which, n - 1, 1, 16).shape == (1, 16)
        with pytest.raises(gm_b200.GmError, match="debug_read"):
            eng.debug_read(which, 0, n + 1, 16)
        with pytest.raises(gm_b200.GmError, match="debug_read"):
            eng.debug_read(which, n, 1, 16)
    torch.cuda.synchronize()
