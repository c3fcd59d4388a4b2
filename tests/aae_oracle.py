"""float64 restatement of the adversarial autoencoder's train step (generative-models_b200/aae.py) - test infrastructure,
numpy only.

One step on a batch x with a given prior sample z_p runs three phases, each on the parameters the one before updated:
recon = sum((x - D(E(x)))^2) with optimizer_R = Adam(encoder + decoder, lr, weight_decay); D_loss =
-mean(log(Dz(z_p) + 1e-8) + log(1 - Dz(E(x)) + 1e-8)) with optimizer_D = Adam(discriminator, D_lr); G_loss =
-mean(log(Dz(E(x)) + 1e-8)) with optimizer_G = Adam(encoder, G_lr), whose moments are its own.  P holds the encoder /
decoder tensors (bir_vae_oracle's names), Dp the discriminator's.  q= and relu= are oracle.ref_math.vae_step's hooks;
relu names: "h1" / "h3" (phase 1 encoder / decoder), "h1d" (the encoder in phases 2 and 3), "hd" (Dz on [z_p ; z_f]),
"hg" (Dz on z_f in phase 3)."""
import numpy as np

from oracle.ref_math import linear, sigmoid, _exact, _relu

ENC = ("encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.mu.bias")
DEC = ("decoder.linear.weight", "decoder.linear.bias", "decoder.recon.weight", "decoder.recon.bias")
DIS = ("discriminator.linear.weight", "discriminator.linear.bias", "discriminator.discriminate.weight",
       "discriminator.discriminate.bias")
LOG_EPS = 1e-8


def encode(P, x, q=_exact, relu=_relu, name="h1"):
    """-> (z = mu(relu(linear(x))), the quantised x, the hidden rows)"""
    xq = q("x", x)
    h1 = q("h", relu(name, linear(xq, q("W", P[ENC[0]]), P[ENC[1]])))
    return linear(h1, q("W", P[ENC[2]]), P[ENC[3]]), xq, h1


def encoder_backward(P, dz, xq, h1, q=_exact):
    """the encoder's gradients from dL/dz"""
    dmu = q("dml", dz)
    da1 = q("da1", (dmu @ q("W", P[ENC[2]])) * (h1 > 0))
    return {ENC[2]: dmu.T @ h1, ENC[3]: dmu.sum(0), ENC[0]: da1.T @ xq, ENC[1]: da1.sum(0)}


def recon_phase(P, x, q=_exact, relu=_relu):
    """-> (recon, gradients of the eight encoder / decoder tensors)"""
    z, xq, h1 = encode(P, x, q, relu)
    zq = q("z", z)
    W3, W4 = q("W", P[DEC[0]]), q("W", P[DEC[2]])
    h3 = q("h", relu("h3", linear(zq, W3, P[DEC[1]])))
    out = sigmoid(linear(h3, W4, P[DEC[3]]))
    recon = np.sum((xq - out) ** 2)
    da4 = q("da4", -2 * (xq - out) * out * (1 - out))
    da3 = q("da3", (da4 @ W4) * (h3 > 0))
    g = {DEC[2]: da4.T @ h3, DEC[3]: da4.sum(0), DEC[0]: da3.T @ zq, DEC[1]: da3.sum(0)}
    g.update(encoder_backward(P, da3 @ W3, xq, h1, q))
    return recon, g


def d_scores(Dp, z, q=_exact, relu=_relu, name="hd"):
    """Dz(z) = sigmoid(discriminate(relu(linear(z)))) -> (scores, logits, the pre-activations, the quantised z)"""
    zq = q("z", z)
    pre = linear(zq, q("W", Dp[DIS[0]]), Dp[DIS[1]])
    a = relu(name, pre)
    s = a @ Dp[DIS[2]][0] + Dp[DIS[3]][0]            # the row-dot runs on the fp32 activations
    return sigmoid(s), s, a, zq


def d_phase(P, Dp, x, prior, q=_exact, relu=_relu):
    """-> (D_loss, gradients of the four discriminator tensors, z_f)"""
    z_f, _, _ = encode(P, x, q, relu, "h1d")
    B = x.shape[0]
    zz = np.concatenate([prior, z_f])
    d, _, a, zq = d_scores(Dp, zz, q, relu, "hd")
    real, fake = d[:B], d[B:]
    loss = -np.mean(np.log(real + LOG_EPS) + np.log(1 - fake + LOG_EPS))
    dd = np.concatenate([-1.0 / (real + LOG_EPS), 1.0 / (1 - fake + LOG_EPS)]) / B
    ds = dd * d * (1 - d)                            # dL/dlogit
    aq = q("h", a)
    dh = q("dh", ds[:, None] * Dp[DIS[2]][0][None, :] * (aq > 0))
    g = {DIS[0]: dh.T @ zq, DIS[1]: dh.sum(0), DIS[2]: (ds[:, None] * aq).sum(0)[None, :], DIS[3]: np.array([ds.sum()])}
    return loss, g, z_f


def g_phase(P, Dp, x, q=_exact, relu=_relu):
    """-> (G_loss, gradients of the four encoder tensors)"""
    z_f, xq, h1 = encode(P, x, q, relu, "h1d")
    B = x.shape[0]
    d, _, a, _ = d_scores(Dp, z_f, q, relu, "hg")
    loss = -np.mean(np.log(d + LOG_EPS))
    ds = -1.0 / (d + LOG_EPS) / B * d * (1 - d)
    M = q("m", Dp[DIS[2]][0][None, :] * (a > 0))
    dz = ds[:, None] * (M @ q("W", Dp[DIS[0]]))
    return loss, encoder_backward(P, dz, xq, h1, q)


def adam(p, g, st, step, lr, wd=0.0, b1=0.9, b2=0.999, eps=1e-8):
    """one torch.optim.Adam update (coupled weight decay) of p with gradient g; st = (m, v), updated in place"""
    g = g + wd * p
    m, v = st
    m[...] = b1 * m + (1 - b1) * g
    v[...] = b2 * v + (1 - b2) * g * g
    return p - lr / (1 - b1 ** step) * (m / (np.sqrt(v) / np.sqrt(1 - b2 ** step) + eps))


def new_state(P, Dp):
    """the three optimizers' moments: R over encoder + decoder, D over the discriminator, G over the encoder"""
    z = lambda names, src: {k: (np.zeros_like(src[k]), np.zeros_like(src[k])) for k in names}
    return dict(R=z(ENC + DEC, P), D=z(DIS, Dp), G=z(ENC, P), steps=[0, 0, 0])


def aae_step(P, Dp, st, x, prior, lr=1e-3, D_lr=2e-4, G_lr=2e-4, weight_decay=1e-5, q=_exact, relu=_relu):
    """one train step: -> (recon, D_loss, G_loss, P, Dp, the three phases' gradients); P / Dp are new dicts, st is updated"""
    P, Dp = dict(P), dict(Dp)
    recon, gr = recon_phase(P, x, q, relu)
    st["steps"][0] += 1
    for k in ENC + DEC:
        P[k] = adam(P[k], gr[k], st["R"][k], st["steps"][0], lr, weight_decay)
    dl, gd, _ = d_phase(P, Dp, x, prior, q, relu)
    st["steps"][1] += 1
    for k in DIS:
        Dp[k] = adam(Dp[k], gd[k], st["D"][k], st["steps"][1], D_lr)
    gl, gg = g_phase(P, Dp, x, q, relu)
    st["steps"][2] += 1
    for k in ENC:
        P[k] = adam(P[k], gg[k], st["G"][k], st["steps"][2], G_lr)
    return recon, dl, gl, P, Dp, (gr, gd, gg)
