"""Shared pieces of the MLP engines' GPU tests (GanEngine, InfoGanEngine, VaeEngine): engine construction from the
seeded weights at any (image, hidden, z) geometry, the gradient-penalty draws, the norm-relative error, and the context
manager that gives near-kink ReLU units the device's side in the numpy oracle."""
import numpy as np
import torch

from inputs import gm_init_weights
from oracle import ref_math as R


def nrel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def gan_shapes(X, H, Z, began=False):
    if began:
        return [("G.linear", (H, Z)), ("G.generate", (X, H)), ("D.encoder", (H, X)), ("D.decoder", (X, H))]
    return [("G.linear", (H, Z)), ("G.generate", (X, H)), ("D.linear", (H, X)), ("D.discriminate", (1, H))]


def gan_engine(variant, X=784, H=400, Z=20, max_batch=64, precision="bf16", seed=1234):
    """GanEngine at (X, H, Z) holding gm_init_weights(seed); D ends in ReLU for WGAN-GP, in a sigmoid otherwise."""
    import gm_b200
    eng = gm_b200.GanEngine(X, H, Z, max_batch=max_batch, variant=variant,
                            d_out_act="relu" if variant == "wgp" else "sigmoid", precision=precision)
    W = gm_init_weights(gan_shapes(X, H, Z, variant == "began"), seed)
    names = list(W)
    eng.load(0, [W[names[0]][0], W[names[0]][1], W[names[1]][0], W[names[1]][1]])
    eng.load(1, [W[names[2]][0], W[names[2]][1], W[names[3]][0], W[names[3]][1]])
    return eng


def aux_from(draws_iter, case):
    """(oracle aux, device aux tensor) for the gradient-penalty variants, consuming draws: WGAN-GP's eps [B,1], DRAGAN's
    (delta [B,1], u [B,X])."""
    if case == "wgp":
        eps = next(draws_iter)
        return eps.astype(np.float64), torch.from_numpy(eps.reshape(-1).copy()).cuda()
    if case == "dra":
        delta, u = next(draws_iter), next(draws_iter)
        dev = torch.from_numpy(np.concatenate([delta.reshape(-1), u.reshape(-1)])).cuda()
        return (delta.astype(np.float64), u.astype(np.float64)), dev
    return None, None


# ReLU boundaries.  dReLU/da is discontinuous at a = 0: a hidden unit whose pre-activation is ~1e-6 (fp32 rounding
# level of a 784-term dot product) lands on either side depending on the summation order - the reference itself flips
# such units between BLAS thread counts (SURVEY.md 8c: 8 vs 1 thread differ at 3e-7) - and one flipped unit moves a
# batch-64 gradient by ~1e-2.  For units with |a| < TOL_A the oracle therefore takes the side the device took (read
# back from the engine's activation buffers); every other unit must agree by itself.  The number of such units is
# reported (0 or 1 per step at these sizes).
TOL_A = 2e-5


class DeviceReluSides:
    """Context manager: patches oracle.ref_math's forward functions so that near-boundary ReLU units take the
    device's side.  d_regions: row offsets (in units of B) of the D-hidden rows for successive d_forward calls.
    fake_rows: row offset (in units of B) of G's output in Xall; when given, G's output is taken as the device stored
    it.  With bf16 storage a fake element whose fp32 and float64 values straddle a rounding boundary differs by one
    bf16 ulp (~2e-3), which moves D's pre-activation on that row by ~1e-4, beyond TOL_A; the model is evaluated at the
    device's storage point instead, after checking that every stored element is within one ulp of the model's."""

    def __init__(self, eng, d_regions, g_hidden=True, fake_rows=None):
        self.eng, self.d_regions, self.g_hidden, self.count = eng, list(d_regions), g_hidden, 0
        self.fake_rows, self.fake_flips = fake_rows, 0

    def __enter__(self):
        self._d, self._g, self._calls = R.d_forward, R.g_forward, 0

        def d_forward(P, x, *a, **k):
            fw = self._d(P, x, *a, **k)
            reg = self.d_regions[min(self._calls, len(self.d_regions) - 1)]
            reg = reg if isinstance(reg, tuple) else ("Aall", reg)
            buf, reg, positive = reg if len(reg) == 3 else (reg[0], reg[1], False)
            self._calls += 1
            near = np.abs(fw["a1"]) < TOL_A
            if near.any():
                n = fw["a1"].shape[0]
                # the buffers hold activations or the signed mask form w2 * relu'(a) (nonzero <=> active); WGAN-GP's real /
                # fake rows hold PRE-activations (positive <=> active; regions flagged `positive`)
                v = self.eng.debug_read(buf, reg * n, n, fw["a1"].shape[1]).cpu().numpy()
                act = (v > 0) if positive else (v != 0)
                for key in ("h", "hq"):
                    v = fw[key].copy()
                    v[near] = np.where(act[near], 1e-30, 0.0)
                    fw[key] = v
                self.count += int(near.sum())
            return fw

        def g_forward(P, z, *a, **k):
            fw = self._g(P, z, *a, **k)
            near = np.abs(fw["a1"]) < TOL_A
            if self.g_hidden and near.any():
                n = fw["a1"].shape[0]
                act = self.eng.debug_read("Hg", 0, n, fw["a1"].shape[1]).cpu().numpy() > 0
                v = fw["h"].copy()
                v[near] = np.where(act[near], 1e-30, 0.0)
                fw["h"] = v
                self.count += int(near.sum())
            if self.fake_rows is not None:
                n, x = fw["out"].shape
                dev = self.eng.debug_read("Xall", self.fake_rows * n, n, x).cpu().numpy().astype(np.float64)
                off = np.abs(dev - fw["out"]) > 2.0 ** -7 * np.abs(fw["out"])
                assert not off.any(), ("stored fake rows beyond one bf16 ulp of the model", int(off.sum()))
                self.fake_flips += int(np.count_nonzero(dev != fw["out"]))
                fw["out"] = dev
            return fw
        R.d_forward, R.g_forward = d_forward, g_forward
        return self

    def __exit__(self, *exc):
        R.d_forward, R.g_forward = self._d, self._g
        return False


class VaeReluSides:
    """relu hook for oracle.ref_math.vae_step: encoder ("h1") and decoder ("h3") hidden units with |a| < TOL_A take the
    side the device took in its last VaeEngine.grad (read back from H1 / H3).  In split mode z is stored as a hi + lo
    bf16 pair (~2^-17 relative), which moves the decoder's pre-activations by ~1e-5 against the exact oracle: about one
    of the 130 000 decoder units of a batch of 300 at H = 432 lands within that of zero."""

    BUF = {"h1": "H1", "h3": "H3"}

    def __init__(self, eng):
        self.eng, self.count = eng, 0

    def __call__(self, name, a):
        h = np.maximum(a, 0)
        near = np.abs(a) < TOL_A
        if near.any():
            n, c = a.shape
            act = self.eng.debug_read(self.BUF[name], 0, n, c).cpu().numpy() > 0
            h[near] = np.where(act[near], 1e-30, 0.0)
            self.count += int(near.sum())
        return h
