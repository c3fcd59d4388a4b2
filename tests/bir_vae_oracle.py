"""float64 restatement of the BIR-VAE train step (src/bir_vae.py:84-95,178-211) - test infrastructure, numpy only.

bir_vae_step takes the same q= (operand-quantisation) and relu= hooks as oracle.ref_math.vae_step; mmd / mmd_grad are
the closed forms the CUDA MMD kernel is checked against."""
import numpy as np

from oracle.ref_math import linear, sigmoid, _exact, _relu


def gauss_kernel(a, b):
    """k(a_i, b_j) = exp(-mean((a_i - b_j)^2) / Z) = exp(-|a_i - b_j|^2 / Z^2)  (src/bir_vae.py:199-211)"""
    Z = a.shape[1]
    d2 = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    return np.exp(-d2 / (Z * Z))


def mmd(z, p, lam=1.0):
    """lam (sum k(p,p) + sum k(z,z) - 2 sum k(p,z))  (src/bir_vae.py:190-197)"""
    return lam * (gauss_kernel(p, p).sum() + gauss_kernel(z, z).sum() - 2 * gauss_kernel(p, z).sum())


def mmd_grad(z, p, lam=1.0):
    """d mmd / dz_i = lam 4/Z^2 (-sum_j k(z_i,z_j)(z_i - z_j) + sum_j k(z_i,p_j)(z_i - p_j))"""
    Z = z.shape[1]
    kzz, kzp = gauss_kernel(z, z), gauss_kernel(z, p)
    t = -(kzz.sum(1)[:, None] * z - kzz @ z) + (kzp.sum(1)[:, None] * z - kzp @ p)
    return lam * 4.0 / (Z * Z) * t


def bir_vae_step(P, x, eps, prior, lam=1000.0, q=_exact, relu=_relu):
    """BIRVAE.forward + compute_batch + backward of mse + mmd: z = mu + eps, mse = sum((x - out)^2),
    mmd = lam * MMD(z, prior).  Returns (mse, mmd, grads of the eight tensors, dict(out, mu, z)).
    q: the CUDA engine's bf16 storage points (weights, x, hidden rows, z, da4, da3, dmu, da1); mu, z for the MMD, dz and
    the losses stay fp32-grade."""
    W1, b1 = q("W", P["encoder.linear.weight"]), P["encoder.linear.bias"]
    Wm, bm = q("W", P["encoder.mu.weight"]), P["encoder.mu.bias"]
    W3, b3 = q("W", P["decoder.linear.weight"]), P["decoder.linear.bias"]
    W4, b4 = q("W", P["decoder.recon.weight"]), P["decoder.recon.bias"]
    xq = q("x", x)
    h1 = q("h", relu("h1", linear(xq, W1, b1)))
    mu = linear(h1, Wm, bm)
    z = mu + eps                                           # src/bir_vae.py:94
    zq = q("z", z)
    h3 = q("h", relu("h3", linear(zq, W3, b3)))
    out = sigmoid(linear(h3, W4, b4))
    mse = np.sum((xq - out) ** 2)
    m = mmd(z, prior, lam)
    g = {}
    da4 = q("da4", -2 * (xq - out) * out * (1 - out))
    g["decoder.recon.weight"] = da4.T @ h3
    g["decoder.recon.bias"] = da4.sum(0)
    da3 = q("da3", (da4 @ W4) * (h3 > 0))
    g["decoder.linear.weight"] = da3.T @ zq
    g["decoder.linear.bias"] = da3.sum(0)
    dmu = q("dml", da3 @ W3 + mmd_grad(z, prior, lam))
    g["encoder.mu.weight"] = dmu.T @ h1
    g["encoder.mu.bias"] = dmu.sum(0)
    da1 = q("da1", (dmu @ Wm) * (h1 > 0))
    g["encoder.linear.weight"] = da1.T @ xq
    g["encoder.linear.bias"] = da1.sum(0)
    return mse, m, g, dict(out=out, mu=mu, z=z)
