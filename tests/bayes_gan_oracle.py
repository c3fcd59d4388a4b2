"""float64 restatement of one Bayesian GAN step (generative-models_b200/bayes_gan.py) - test infrastructure, numpy only,
built on oracle.ref_math's g_forward / d_forward / d_backward / g_backward.

PG is a list of J generator parameter dicts ("G.linear.weight", ... as in ref_math), PD the discriminator's ("D.*").
Each generator j reads its own noise rows zs[j] [B, z].  The energies (NS, sigmoid D output):
  U_D = -mean_i log(D(x_i) + 1e-8) - mean_{j,i} log(1 - D(G_j(z_ji)) + 1e-8)
  U_j = -mean_i log(D(G_j(z_ji)) + 1e-8), reported as mean_j U_j
and SGHMC with a given xi:
  v <- (1 - alpha) v - lr (g + theta / (prior_std^2 N)) + sqrt(2 alpha lr / N) xi,  theta <- theta + v
q= is ref_math's operand-quantisation hook; fakes= (optional, one [B, X] array per sample) evaluates D at given fake
images (the device's stored bf16 values) instead of the model's."""
import numpy as np

from oracle import ref_math as R

EPS = 1e-8
G_KEYS = ("G.linear.weight", "G.linear.bias", "G.generate.weight", "G.generate.bias")
D_KEYS = ("D.linear.weight", "D.linear.bias", "D.discriminate.weight", "D.discriminate.bias")


def d_step(PG, PD, x, zs, q=R._exact, fakes=None):
    """-> (U_D, D's gradients, the D outputs [real; fake_1; ...; fake_J])"""
    J, B = len(PG), x.shape[0]
    fx = R.d_forward(PD, x, q=q)
    gx, _ = R.d_backward(PD, fx, R.d_out_grad(fx, -1 / (B * (fx["d"] + EPS)), "sigmoid"), q=q)
    loss = -np.mean(np.log(fx["d"] + EPS))
    grads = dict(gx)
    outs = [fx["d"]]
    for j in range(J):
        fake = R.g_forward(PG[j], zs[j], q=q)["out"] if fakes is None else fakes[j]
        fg = R.d_forward(PD, fake, q=q)
        loss += -np.mean(np.log(1 - fg["d"] + EPS)) / J
        gg, _ = R.d_backward(PD, fg, R.d_out_grad(fg, 1 / (J * B * ((1 - fg["d"]) + EPS)), "sigmoid"), q=q)
        grads = {k: grads[k] + gg[k] for k in grads}
        outs.append(fg["d"])
    return loss, grads, np.concatenate(outs)


def g_step(PG, PD, zs, q=R._exact, fakes=None):
    """-> (mean_j U_j, [sample j's gradients of U_j], [U_j])"""
    losses, grads = [], []
    for j in range(len(PG)):
        gf = R.g_forward(PG[j], zs[j], q=q)
        if fakes is not None:
            gf["out"] = fakes[j]
        fg = R.d_forward(PD, gf["out"], q=q)
        L, ddg = R.g_loss("ns", fg["d"])
        _, dxg = R.d_backward(PD, fg, R.d_out_grad(fg, ddg, "sigmoid"), need_dx=True, q=q)
        losses.append(L)
        grads.append(R.g_backward(PG[j], gf, dxg, q=q))
    return float(np.mean(losses)), grads, losses


def sghmc(theta, v, g, xi, lr, alpha, prior_std, data_size):
    """one SGHMC update -> (theta, v), float64"""
    v = (1 - alpha) * v - lr * (g + theta / (prior_std ** 2 * data_size)) + np.sqrt(2 * alpha * lr / data_size) * xi
    return theta + v, v
