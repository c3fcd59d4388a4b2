"""CPU oracle — TEST INFRASTRUCTURE, not product code.

A plain-numpy restatement (closed-form forward, backward and Adam; no autograd,
no torch) of the reference's train-step hot path.  Only tests/, bench.py's
cpu_baseline / --impl reference leg and __graft_entry__.smoke() may import it; the
product path (generative-models_b200/) never does and fails loudly without its
CUDA library.

Parity status: PINNED.  tests/test_oracle_golden.py checks every function here
against tests/golden/*.npz, which tests/golden/make_golden.py produced by running
the unmodified reference (/root/reference/src/*.py on torch 2.11 CPU) in the
build container.  The reference itself ships no golden vectors (SURVEY.md 8c).

Every function cites the reference lines it restates (paths relative to
/root/reference/).  dtype is a parameter: float32 reproduces the reference's
arithmetic type, float64 is used as the high-precision yardstick.
"""
import numpy as np

EPS = 1e-8  # the reference's log-stabiliser, e.g. src/ns_gan.py:191


# ---------------------------------------------------------------- primitives
def bf16_round(x):
    """Round-to-nearest-even to bfloat16, returned in x's dtype (what the CUDA path
    stores for GEMM operands)."""
    a = np.asarray(x, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(np.float32).astype(np.asarray(x).dtype)


def _exact(name, v):
    return v


def bf16_points(name, v):
    """Quantisation hook modelling the CUDA bf16 path: every tensor that is a
    tensor-core GEMM operand (weights, z, hidden, fake, dh, da2, dhg) is bf16;
    biases, the 400->1 row-dot, losses and all accumulation stay fp32."""
    return bf16_round(v)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def linear(x, W, b):
    """nn.Linear: x @ W.T + b  (src/ns_gan.py:40-41)."""
    return x @ W.T + b


def g_forward(P, z, pre="G.", q=_exact):
    """Generator.forward, src/ns_gan.py:43-46: sigmoid(W2 relu(W1 z + b1) + b2).
    q: optional operand-quantisation hook (bf16_points models the CUDA path)."""
    z = q("z", z)
    a1 = linear(z, q("W", P[pre + "linear.weight"]), P[pre + "linear.bias"])
    h = q("h", np.maximum(a1, 0))
    a2 = linear(h, q("W", P[pre + "generate.weight"]), P[pre + "generate.bias"])
    return dict(z=z, a1=a1, h=h, a2=a2, out=q("fake", sigmoid(a2)))


def d_forward(P, x, out_act="sigmoid", pre="D.", q=_exact):
    """Discriminator.forward, src/ns_gan.py:57-60 (sigmoid out);
    src/w_gp_gan.py:59-62 (ReLU out)."""
    a1 = linear(x, q("W", P[pre + "linear.weight"]), P[pre + "linear.bias"])
    h = np.maximum(a1, 0)
    s = linear(h, P[pre + "discriminate.weight"], P[pre + "discriminate.bias"])  # [B,1]
    if out_act == "sigmoid":
        d = sigmoid(s)
    elif out_act == "relu":
        d = np.maximum(s, 0)
    else:
        d = s
    return dict(x=x, a1=a1, h=h, hq=q("a", h), s=s, d=d)


def d_out_grad(fw, dd, out_act):
    """dL/ds from dL/dd through D's last activation."""
    if out_act == "sigmoid":
        return dd * fw["d"] * (1 - fw["d"])
    if out_act == "relu":
        return dd * (fw["s"] > 0)
    return dd


def d_backward(P, fw, ds, need_dx=False, pre="D.", q=_exact):
    """Backward of the 2-layer D from dL/ds [B,1] (autograd of src/ns_gan.py:57-60;
    ReLU' = 0 at 0 like torch's threshold_backward)."""
    W1 = P[pre + "linear.weight"]
    w2 = P[pre + "discriminate.weight"]
    g = {}
    g[pre + "discriminate.weight"] = ds.T @ fw["hq"]
    g[pre + "discriminate.bias"] = ds.sum(0)
    dh = q("dh", (ds @ w2) * (fw["hq"] > 0))
    g[pre + "linear.weight"] = dh.T @ fw["x"]
    g[pre + "linear.bias"] = dh.sum(0)
    # dL/dx: the CUDA G step forms M = w2 * relu'(a1) as the bf16 GEMM operand and applies
    # the per-row factor ds in fp32 after the product (same value; different rounding point)
    dx = ds * (q("mw", w2 * (fw["hq"] > 0)) @ q("W", W1)) if need_dx else None
    return g, dx


def g_backward(P, fw, dout, pre="G.", q=_exact):
    """Backward of G from dL/d(out) [B,X] (autograd of src/ns_gan.py:43-46)."""
    da2 = q("da2", dout * fw["out"] * (1 - fw["out"]))
    g = {}
    g[pre + "generate.weight"] = da2.T @ fw["h"]
    g[pre + "generate.bias"] = da2.sum(0)
    dh = q("dhg", (da2 @ q("W", P[pre + "generate.weight"])) * (fw["h"] > 0))
    g[pre + "linear.weight"] = dh.T @ fw["z"]
    g[pre + "linear.bias"] = dh.sum(0)
    return g


# ---------------------------------------------------------------- loss table
# SURVEY.md Appendix A.1; each entry returns (loss, dL/d dx, dL/d dg) for the D
# step or (loss, dL/d dg) for the G step.  dx, dg are D's outputs [B,1].
D_OUT_ACT = {"wgp": "relu"}


def d_loss(variant, dx, dg, st=None):
    B = dx.shape[0]
    one = dx.dtype.type(1)
    if variant in ("ns", "mm", "dra", "info"):
        # src/ns_gan.py:191-192, src/mm_gan.py:215-216, src/dra_gan.py:195-196
        L = -np.mean(np.log(dx + EPS) + np.log(one - dg + EPS))
        return L, -1 / (B * (dx + EPS)), 1 / (B * ((one - dg) + EPS))
    if variant in ("w", "wgp"):
        # src/w_gan.py:208 ; src/w_gp_gan.py:218 (GP added by caller)
        L = np.mean(dg) - np.mean(dx)
        return L, -np.ones_like(dx) / B, np.ones_like(dg) / B
    if variant == "ls":
        # src/ls_gan.py:192-193 (a=0, b=1)
        L = 0.5 * np.mean((dx - 1) ** 2) + 0.5 * np.mean(dg ** 2)
        return L, (dx - 1) / B, dg / B
    if variant == "ra":
        # src/ra_gan.py:204-205 (code, not docstring)
        m = np.mean(dg)
        q = sigmoid(dx - m)
        r = sigmoid(1 - dg)
        L = -np.mean(np.log(q + EPS) + np.log(r + EPS)) / 2
        gq = q * (1 - q) / (q + EPS)
        gx = -gq / (2 * B)
        gg = (np.sum(gq) / B + r * (1 - r) / (r + EPS)) / (2 * B)
        return L, gx, gg
    if variant == "fisher":
        # src/fisher_gan.py:214-223 ; st = dict(LAMBDA, RHO)
        lam, rho = st["LAMBDA"], st["RHO"]
        m1x, m1g = np.mean(dx), np.mean(dg)
        m2x, m2g = np.mean(dx ** 2), np.mean(dg ** 2)
        om = 1 - (0.5 * m2x + 0.5 * m2g)
        L = -((m1x - m1g) + lam * om - (rho / 2) * om ** 2)
        c = lam - rho * om
        st["dLAMBDA"] = -om
        return L, -(1 - c * dx) / B, (1 + c * dg) / B
    if variant.startswith("f_"):
        # src/f_gan.py:99-121
        m = variant[2:]
        if m == "total_variation":
            L = -(np.mean(0.5 * np.tanh(dx)) - np.mean(0.5 * np.tanh(dg)))
            return L, -0.5 * (1 - np.tanh(dx) ** 2) / B, 0.5 * (1 - np.tanh(dg) ** 2) / B
        if m == "forward_kl":
            L = -(np.mean(dx) - np.mean(np.exp(dg - 1)))
            return L, -np.ones_like(dx) / B, np.exp(dg - 1) / B
        if m == "reverse_kl":
            L = -(np.mean(-np.exp(dx)) - np.mean(-1 - dg))
            return L, np.exp(dx) / B, -np.ones_like(dg) / B
        if m == "pearson":
            L = -(np.mean(dx) - np.mean(0.25 * dg ** 2 + dg))
            return L, -np.ones_like(dx) / B, (0.5 * dg + 1) / B
        if m == "hellinger":
            L = -(np.mean(1 - np.exp(dx)) - np.mean((1 - np.exp(dg)) / np.exp(dg)))
            return L, np.exp(dx) / B, -np.exp(-dg) / B
        if m == "jensen_shannon":
            L = -(np.mean(2 - (1 + np.exp(-dx))) - np.mean(-(2 - np.exp(dg))))
            return L, -np.exp(-dx) / B, np.exp(dg) / B
    raise ValueError(variant)


def g_loss(variant, dg):
    B = dg.shape[0]
    one = dg.dtype.type(1)
    if variant in ("ns", "dra", "ra", "info"):
        # src/ns_gan.py:214 ; src/dra_gan.py:243 ; src/ra_gan.py:227
        return -np.mean(np.log(dg + EPS)), -1 / (B * (dg + EPS))
    if variant == "mm":
        # src/mm_gan.py:235
        return np.mean(np.log((one - dg) + EPS)), -1 / (B * ((one - dg) + EPS))
    if variant in ("w", "wgp", "fisher"):
        # src/w_gan.py:227 ; src/w_gp_gan.py:237 ; src/fisher_gan.py:246
        return -np.mean(dg), -np.ones_like(dg) / B
    if variant == "ls":
        # src/ls_gan.py:213 (c=1)
        return 0.5 * np.mean((dg - 1) ** 2), (dg - 1) / B
    if variant.startswith("f_"):
        # src/f_gan.py:123-142
        m = variant[2:]
        if m == "total_variation":
            return -np.mean(0.5 * np.tanh(dg)), -0.5 * (1 - np.tanh(dg) ** 2) / B
        if m == "forward_kl":
            return -np.mean(np.exp(dg - 1)), -np.exp(dg - 1) / B
        if m == "reverse_kl":
            return -np.mean(-1 - dg), np.ones_like(dg) / B
        if m == "pearson":
            return -np.mean(0.25 * dg ** 2 + dg), -(0.5 * dg + 1) / B
        if m == "hellinger":
            return -np.mean((1 - np.exp(dg)) / np.exp(dg)), np.exp(-dg) / B
        if m == "jensen_shannon":
            return -np.mean(-(2 - np.exp(dg))), -np.exp(dg) / B
    raise ValueError(variant)


# ---------------------------------------------------------------- gradient penalty
def gradient_penalty(P, xhat, out_act, lam=10.0, K=1.0, pre="D.", q=_exact, a1=None):
    """lam * mean((||d D(xhat)/d xhat||_2 - K)^2) and its gradient w.r.t. D's
    parameters, in closed form (SURVEY.md A.2).  Restates
    src/w_gp_gan.py:201-215 (out_act='relu') and src/dra_gan.py:208-220
    (out_act='sigmoid'); norm subgradient 0 at 0 like torch's norm backward.
    q: operand-quantisation hook (bf16_points models the CUDA path).
    a1: the hidden pre-activation of the xhat rows when the caller already has it (the CUDA WGAN-GP path never forms
    xhat: the first layer is linear, a1(xhat) = eps a1(x) + (1-eps) a1(G(z)), gm_b200 gp_hat_kernel); with q = identity
    this is the same number as linear(xhat, W1, b1)."""
    W1, b1 = P[pre + "linear.weight"], P[pre + "linear.bias"]
    w2 = P[pre + "discriminate.weight"]
    if a1 is None:
        xhat = q("xhat", xhat)
        fw = d_forward(P, xhat, out_act, pre, q=q)
    else:
        h = np.maximum(a1, 0)
        s_ = linear(h, w2, P[pre + "discriminate.bias"])
        d_ = sigmoid(s_) if out_act == "sigmoid" else (np.maximum(s_, 0) if out_act == "relu" else s_)
        fw = dict(x=xhat, a1=a1, h=h, hq=h, s=s_, d=d_)
    B = xhat.shape[0]
    M = (fw["hq"] > 0).astype(xhat.dtype)
    if out_act == "relu":
        qq = (fw["s"] > 0).astype(xhat.dtype)        # [B,1]
        dq_ds = np.zeros_like(qq)
    else:
        p = fw["d"]
        qq = p * (1 - p)
        dq_ds = qq * (1 - 2 * p)
    U = q("dh", M * w2)                              # [B,H]
    V = U @ q("W", W1)                               # [B,X]
    nv = np.sqrt(np.sum(V * V, axis=1, keepdims=True))
    V = q("V", V)
    n = qq * nv                                      # = ||q V||, q >= 0
    gp = lam * np.mean((n - K) ** 2)
    r = (2 * lam / B) * (n - K)                      # dGP/dn  [B,1]
    safe = np.where(nv > 0, nv, 1)
    coef = np.where(nv > 0, r * qq / safe, 0)            # dGP/dV = coef * V  [B,1]
    # the CUDA path never forms R = coef * V: it scales the smaller U rows (dGP/dW1 = (coef U)^T V) and applies coef
    # as a per-row factor in the epilogue of T's GEMM; with q = identity this is the same arithmetic
    Us = q("dh", coef * U)
    g = {}
    g[pre + "linear.weight"] = Us.T @ V
    T = q("T", coef * (V @ q("W", W1).T) * M)
    g[pre + "discriminate.weight"] = np.sum(T, axis=0, keepdims=True)
    g[pre + "linear.bias"] = np.zeros_like(b1)
    g[pre + "discriminate.bias"] = np.zeros(1, dtype=xhat.dtype)
    # path through q(s) (sigmoid out only)
    ds = r * nv * dq_ds
    if np.any(ds != 0):
        g2, _ = d_backward(P, fw, ds, pre=pre, q=q)
        for k in g:
            g[k] = g[k] + g2[k].reshape(g[k].shape)
    return gp, g, dict(n=n, fw=fw)


# ---------------------------------------------------------------- train steps
def gan_d_step(P, variant, images, z, aux=None, st=None, lam=10.0, q=_exact, pre_points=None):
    """Trainer.train_D + D_loss.backward(), restricted to D's gradients (the G
    gradients the reference also computes are discarded at src/ns_gan.py:148).
    aux: for 'wgp' eps [B,1] (src/w_gp_gan.py:197); for 'dra' (delta [B,1],
    u [B,X]) (src/dra_gan.py:200,205).
    pre_points: (a1 of the real rows, a1 of the fake rows) as STORED by the device (bf16), for 'wgp' with a quantising q:
    the model is then evaluated at the device's storage points (a 1-ulp difference in a stored pre-activation - fp32
    vs float64 accumulation order - moves a_hat by ~1e-3 and can flip a near-zero unit of the penalty's mask)."""
    act = D_OUT_ACT.get(variant, "sigmoid")
    gf = g_forward(P, z, q=q)
    fx = d_forward(P, images, act, q=q)
    fg = d_forward(P, gf["out"], act, q=q)
    L, ddx, ddg = d_loss(variant, fx["d"], fg["d"], st)
    gx, _ = d_backward(P, fx, d_out_grad(fx, ddx, act), q=q)
    gg, _ = d_backward(P, fg, d_out_grad(fg, ddg, act), q=q)
    grads = {k: gx[k] + gg[k] for k in gx}
    info = dict(dx=fx["d"], dg=fg["d"], fake=gf["out"])
    if variant == "wgp":
        eps = aux
        xhat = eps * images + (1 - eps) * gf["out"]                   # src/w_gp_gan.py:201
        # the bf16-point model follows the CUDA path: pre-activations of the real / fake rows are stored (rounded), the
        # xhat rows are not formed
        if q is _exact:
            a1h = None
        elif pre_points is not None:
            a1h = eps * pre_points[0] + (1 - eps) * pre_points[1]
        else:
            a1h = eps * q("a", fx["a1"]) + (1 - eps) * q("a", fg["a1"])
        gp, ggp, gi = gradient_penalty(P, xhat, "relu", lam=lam, q=q, a1=a1h)
        L = L + gp
        grads = {k: grads[k] + ggp[k].reshape(grads[k].shape) for k in grads}
        info.update(gp=gp, gp_n=gi["n"])
    if variant == "dra":
        delta, u = aux
        std = np.std(images.astype(np.float64), ddof=1).astype(images.dtype)  # images.std(): unbiased, global
        xhat = delta * images + (1 - delta) * (images + std * u)      # src/dra_gan.py:203-205 (C=1)
        gp, ggp, gi = gradient_penalty(P, xhat, "sigmoid", lam=lam, q=q)
        L = L + gp
        grads = {k: grads[k] + ggp[k].reshape(grads[k].shape) for k in grads}
        info.update(gp=gp, gp_n=gi["n"])
    return L, grads, info


def gan_g_step(P, variant, z, q=_exact):
    """Trainer.train_G + G_loss.backward(), restricted to G's gradients
    (src/ns_gan.py:196-216,155)."""
    act = D_OUT_ACT.get(variant, "sigmoid")
    gf = g_forward(P, z, q=q)
    fg = d_forward(P, gf["out"], act, q=q)
    L, ddg = g_loss(variant, fg["d"])
    _, dxg = d_backward(P, fg, d_out_grad(fg, ddg, act), need_dx=True, q=q)
    return L, g_backward(P, gf, dxg, q=q), dict(dg=fg["d"], fake=gf["out"])


class Adam:
    """torch.optim.Adam (torch 2.11 single-tensor form) as used at
    src/ns_gan.py:107-110 and src/vae.py:139-142 (coupled weight decay):
    g += wd*p; m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2;
    p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)."""

    def __init__(self, keys, lr, b1=0.9, b2=0.999, eps=1e-8, wd=0.0):
        self.keys, self.lr, self.b1, self.b2, self.eps, self.wd = list(keys), lr, b1, b2, eps, wd
        self.t, self.m, self.v = 0, {}, {}

    def step(self, P, grads):
        self.t += 1
        for k in self.keys:
            p = P[k]
            dt = p.dtype.type
            g = grads[k].reshape(p.shape).astype(p.dtype)
            if self.wd:
                g = g + dt(self.wd) * p
            m = self.m.get(k, np.zeros_like(p))
            v = self.v.get(k, np.zeros_like(p))
            m = dt(self.b1) * m + dt(1 - self.b1) * g
            v = dt(self.b2) * v + dt(1 - self.b2) * g * g
            bc1 = 1 - self.b1 ** self.t
            bc2 = 1 - self.b2 ** self.t
            denom = np.sqrt(v) / dt(np.sqrt(bc2)) + dt(self.eps)
            P[k] = p - dt(self.lr / bc1) * (m / denom)
            self.m[k], self.v[k] = m, v


def gan_train(P, variant, images, draws, steps, G_lr, D_lr, D_steps=1, clip=None,
              G_init=0, RHO=1e-6, lam=10.0):
    """The Trainer.train inner loop (src/ns_gan.py:122-156) with the variant
    extras: MM G pre-steps (src/mm_gan.py:121-136), WGAN clamp after each D step
    (src/w_gan.py:158), Fisher lambda update between backward and step
    (src/fisher_gan.py:152-159).  `draws` is an iterator over the recorded RNG
    tensors in the reference's call order."""
    draws = iter(draws)
    gk = [k for k in P if k.startswith("G.")]
    dk = [k for k in P if k.startswith("D.")]
    optG, optD = Adam(gk, G_lr), Adam(dk, D_lr)
    st = dict(LAMBDA=images.dtype.type(0), RHO=images.dtype.type(RHO)) if variant == "fisher" else None
    for _ in range(G_init):
        L, g, _ = gan_g_step(P, variant, next(draws))
        optG.step(P, g)
    Dl, Gl = [], []
    for _ in range(steps):
        acc = []
        for _ in range(D_steps):
            z = next(draws)
            aux = None
            if variant == "wgp":
                aux = next(draws)
            if variant == "dra":
                aux = (next(draws), next(draws))
            L, g, _ = gan_d_step(P, variant, images, z, aux, st, lam)
            if variant == "fisher":
                st["LAMBDA"] = st["LAMBDA"] + st["RHO"] * st["dLAMBDA"]
            optD.step(P, g)
            if clip is not None:
                for k in dk:
                    P[k] = np.clip(P[k], -clip, clip)
            acc.append(float(L))
        Dl.append(np.mean(acc))
        L, g, _ = gan_g_step(P, variant, next(draws))
        Gl.append(float(L))
        optG.step(P, g)
    return np.array(Dl), np.array(Gl), st


# ---------------------------------------------------------------- VAE
def _relu(name, a):
    return np.maximum(a, 0)


def vae_step(P, x, eps, q=_exact, relu=_relu):
    """VAE.forward + compute_batch + backward (src/vae.py:94-106,193-212):
    recon = sum((x-out)^2), kl = sum(0.5(mu^2+exp(lv)-lv-1)); returns grads of
    recon+kl for all ten tensors.
    q: operand-quantisation hook at the points where the CUDA VAE stores bf16 GEMM operands (bf16_points models it):
    the weights, x, the hidden rows, z, and the upstream gradients da4, da3, [dmu | dlv], da1; mu / log_var, dz, the
    reconstruction and both losses stay fp32.
    relu: relu(name, a) for the encoder ("h1") and decoder ("h3") hidden layers (tests give near-zero units a side);
    the ReLU masks of the backward are taken from its output."""
    W1, b1 = q("W", P["encoder.linear.weight"]), P["encoder.linear.bias"]
    Wm, bm = q("W", P["encoder.mu.weight"]), P["encoder.mu.bias"]
    Wv, bv = q("W", P["encoder.log_var.weight"]), P["encoder.log_var.bias"]
    W3, b3 = q("W", P["decoder.linear.weight"]), P["decoder.linear.bias"]
    W4, b4 = q("W", P["decoder.recon.weight"]), P["decoder.recon.bias"]
    xq = q("x", x)
    a1 = linear(xq, W1, b1)
    h1 = q("h", relu("h1", a1))
    mu, lv = linear(h1, Wm, bm), linear(h1, Wv, bv)
    sd = np.exp(lv / 2)
    z = q("z", mu + eps * sd)                              # src/vae.py:105
    a3 = linear(z, W3, b3)
    h3 = q("h", relu("h3", a3))
    out = sigmoid(linear(h3, W4, b4))
    recon = np.sum((xq - out) ** 2)                        # src/vae.py:203
    kl = np.sum(0.5 * (mu ** 2 + np.exp(lv) - lv - 1))     # src/vae.py:212
    g = {}
    da4 = q("da4", -2 * (xq - out) * out * (1 - out))
    g["decoder.recon.weight"] = da4.T @ h3
    g["decoder.recon.bias"] = da4.sum(0)
    da3 = q("da3", (da4 @ W4) * (h3 > 0))
    g["decoder.linear.weight"] = da3.T @ z
    g["decoder.linear.bias"] = da3.sum(0)
    dz = da3 @ W3
    dmu = q("dml", mu + dz)
    dlv = q("dml", 0.5 * (np.exp(lv) - 1) + dz * eps * sd * 0.5)
    g["encoder.mu.weight"] = dmu.T @ h1
    g["encoder.mu.bias"] = dmu.sum(0)
    g["encoder.log_var.weight"] = dlv.T @ h1
    g["encoder.log_var.bias"] = dlv.sum(0)
    da1 = q("da1", (dmu @ Wm + dlv @ Wv) * (h1 > 0))
    g["encoder.linear.weight"] = da1.T @ xq
    g["encoder.linear.bias"] = da1.sum(0)
    return recon, kl, g, dict(out=out, mu=mu, lv=lv)


def vae_train(P, x, draws, steps, lr=1e-3, wd=1e-5):
    """VAETrainer.train inner loop (src/vae.py:150-167)."""
    opt = Adam(list(P.keys()), lr, wd=wd)
    R, K = [], []
    for _, eps in zip(range(steps), draws):
        recon, kl, g, _ = vae_step(P, x, eps)
        opt.step(P, g)
        R.append(float(recon))
        K.append(float(kl))
    return np.array(R), np.array(K)


# ---------------------------------------------------------------- InfoGAN (src/info_gan.py)
def info_q_step(P, noise, z_dim=20, disc_dim=10, q=_exact):
    """InfoGANTrainer.train_Q + MI_loss.backward() (src/info_gan.py:269-304): CE on the
    categorical code + MSE on the continuous code (both torch means, LAMBDA = 1); returns
    the loss and the gradients for G and Q."""
    gf = g_forward(P, noise, q=q)
    fake = gf["out"]
    a1 = linear(fake, q("W", P["Q.linear.weight"]), P["Q.linear.bias"])
    hq = q("h", np.maximum(a1, 0))
    inf = linear(hq, q("W", P["Q.inference.weight"]), P["Q.inference.bias"])
    B = noise.shape[0]
    disc, cont = inf[:, :disc_dim], inf[:, disc_dim:]
    tgt = np.argmax(noise[:, z_dim:z_dim + disc_dim], axis=1)
    m = disc.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.sum(np.exp(disc - m), axis=1))
    ce = np.mean(lse - disc[np.arange(B), tgt])
    ctgt = noise[:, z_dim + disc_dim:]
    mse = np.mean((cont - ctgt) ** 2)
    L = ce + mse
    sm = np.exp(disc - lse[:, None])
    sm[np.arange(B), tgt] -= 1
    dinf = q("dinf", np.concatenate([sm / B, 2 * (cont - ctgt) / cont.size], axis=1))
    g = {}
    g["Q.inference.weight"] = dinf.T @ hq
    g["Q.inference.bias"] = dinf.sum(0)
    dhq = q("dh", (dinf @ q("W", P["Q.inference.weight"])) * (hq > 0))
    g["Q.linear.weight"] = dhq.T @ fake
    g["Q.linear.bias"] = dhq.sum(0)
    dfake = dhq @ q("W", P["Q.linear.weight"])
    g.update(g_backward(P, gf, dfake, q=q))
    return L, g


# ---------------------------------------------------------------- BEGAN (src/be_gan.py)
def began_ae(P, x, q=_exact):
    """Discriminator = autoencoder x -> relu(We x + be) -> Wd e + bd (src/be_gan.py:63-76)."""
    a1 = linear(x, q("W", P["D.encoder.weight"]), P["D.encoder.bias"])
    e = q("h", np.maximum(a1, 0))
    r = linear(e, q("W", P["D.decoder.weight"]), P["D.decoder.bias"])
    return dict(x=x, e=e, r=r)


def began_ae_backward(P, fw, dr, q=_exact, need_dx=False):
    dr = q("dr", dr)
    g = {"D.decoder.weight": dr.T @ fw["e"], "D.decoder.bias": dr.sum(0)}
    de = q("dh", (dr @ q("W", P["D.decoder.weight"])) * (fw["e"] > 0))
    g["D.encoder.weight"] = de.T @ fw["x"]
    g["D.encoder.bias"] = de.sum(0)
    return g, (de @ q("W", P["D.encoder.weight"]) if need_dx else None)


def began_d_step(P, x, z, K, q=_exact):
    """train_D + backward (src/be_gan.py:212-238,168-169): D_loss = DX - K*DG with L1
    reconstruction losses; only D's gradients."""
    B = x.shape[0]
    gf = g_forward(P, z, q=q)
    fx, fg = began_ae(P, x, q), began_ae(P, gf["out"], q)
    DX = np.mean(np.sum(np.abs(fx["r"] - x), axis=1))
    DG = np.mean(np.sum(np.abs(fg["r"] - gf["out"]), axis=1))
    gx, _ = began_ae_backward(P, fx, np.sign(fx["r"] - x) / B, q)
    gg, _ = began_ae_backward(P, fg, -K * np.sign(fg["r"] - gf["out"]) / B, q)
    return DX - K * DG, {k: gx[k] + gg[k] for k in gx}, DX, DG


def began_g_step(P, z, q=_exact):
    """train_G + backward (src/be_gan.py:240-258,177-178): G_loss = E sum |D(G(z)) - G(z)|;
    the gradient reaches G(z) both through D and directly."""
    B = z.shape[0]
    gf = g_forward(P, z, q=q)
    fg = began_ae(P, gf["out"], q)
    s = np.sign(fg["r"] - gf["out"]) / B
    L = np.mean(np.sum(np.abs(fg["r"] - gf["out"]), axis=1))
    _, dx = began_ae_backward(P, fg, s, q, need_dx=True)
    return L, g_backward(P, gf, dx - q("dr", s), q=q)


def began_train(P, x, draws, steps, G_lr=1e-4, D_lr=1e-4, GAMMA=0.5, LAMBDA=1e-3, K=0.0):
    """BEGANTrainer.train inner loop (src/be_gan.py:147-195) incl. the proportional control
    of K; the two ReduceLROnPlateau schedulers (patience 5 epochs) are inert over a few steps."""
    draws = iter(draws)
    optG = Adam([k for k in P if k.startswith("G.")], G_lr)
    optD = Adam([k for k in P if k.startswith("D.")], D_lr)
    Dl, Gl = [], []
    for _ in range(steps):
        L, g, DX, DG = began_d_step(P, x, next(draws), K)
        optD.step(P, g)
        Dl.append(float(L))
        Lg, gg = began_g_step(P, next(draws))
        optG.step(P, gg)
        Gl.append(float(Lg))
        K = min(max(0.0, K + LAMBDA * (GAMMA * DX - DG)), 1.0)
    return np.array(Dl), np.array(Gl), K
