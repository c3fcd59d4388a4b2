"""float64 restatement of the conditional VAE train step (generative-models_b200/cvae.py) - test infrastructure, numpy only.

cvae_step takes the same q= (operand-quantisation) and relu= hooks as oracle.ref_math.vae_step.  Each conditional layer
is written as its x (z) product plus its one-hot product, so with zero label columns every value is the one
ref_math.vae_step computes, bit for bit (only exact zeros are added)."""
import numpy as np

from oracle.ref_math import linear, sigmoid, _exact, _relu


def onehot(y, num_classes):
    return np.eye(num_classes)[np.asarray(y)]


def cvae_step(P, x, y, eps, num_classes, q=_exact, relu=_relu):
    """CVAE.forward + compute_batch + backward: encoder on [x | onehot(y)], z = mu + eps exp(lv / 2), decoder on
    [z | onehot(y)], recon = sum((x - out)^2), kl = sum(0.5 (mu^2 + exp(lv) - lv - 1)).  Returns (recon, kl, grads of the
    ten tensors, dict(out, mu, lv, z)).
    q: the CUDA engine's bf16 storage points (weights, x, the hidden rows, z, da4, da3, [dmu | dlv], da1); the one-hot
    columns are exact in bf16."""
    X = x.shape[1]
    Z = P["encoder.mu.weight"].shape[0]
    Y = onehot(y, num_classes)
    W1, b1 = q("W", P["encoder.linear.weight"]), P["encoder.linear.bias"]
    Wm, bm = q("W", P["encoder.mu.weight"]), P["encoder.mu.bias"]
    Wv, bv = q("W", P["encoder.log_var.weight"]), P["encoder.log_var.bias"]
    W3, b3 = q("W", P["decoder.linear.weight"]), P["decoder.linear.bias"]
    W4, b4 = q("W", P["decoder.recon.weight"]), P["decoder.recon.bias"]
    xq = q("x", x)
    a1 = linear(xq, W1[:, :X], b1) + Y @ W1[:, X:].T
    h1 = q("h", relu("h1", a1))
    mu, lv = linear(h1, Wm, bm), linear(h1, Wv, bv)
    sd = np.exp(lv / 2)
    z = q("z", mu + eps * sd)
    a3 = linear(z, W3[:, :Z], b3) + Y @ W3[:, Z:].T
    h3 = q("h", relu("h3", a3))
    out = sigmoid(linear(h3, W4, b4))
    recon = np.sum((xq - out) ** 2)
    kl = np.sum(0.5 * (mu ** 2 + np.exp(lv) - lv - 1))
    g = {}
    da4 = q("da4", -2 * (xq - out) * out * (1 - out))
    g["decoder.recon.weight"] = da4.T @ h3
    g["decoder.recon.bias"] = da4.sum(0)
    da3 = q("da3", (da4 @ W4) * (h3 > 0))
    g["decoder.linear.weight"] = np.concatenate([da3.T @ z, da3.T @ Y], axis=1)
    g["decoder.linear.bias"] = da3.sum(0)
    dz = da3 @ W3[:, :Z]
    dmu = q("dml", mu + dz)
    dlv = q("dml", 0.5 * (np.exp(lv) - 1) + dz * eps * sd * 0.5)
    g["encoder.mu.weight"] = dmu.T @ h1
    g["encoder.mu.bias"] = dmu.sum(0)
    g["encoder.log_var.weight"] = dlv.T @ h1
    g["encoder.log_var.bias"] = dlv.sum(0)
    da1 = q("da1", (dmu @ Wm + dlv @ Wv) * (h1 > 0))
    g["encoder.linear.weight"] = np.concatenate([da1.T @ xq, da1.T @ Y], axis=1)
    g["encoder.linear.bias"] = da1.sum(0)
    return recon, kl, g, dict(out=out, mu=mu, lv=lv, z=z, da1=da1, da3=da3)
