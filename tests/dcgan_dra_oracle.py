"""DRAGAN conv discriminator oracle — test infrastructure, not product code.

The batch-norm-free critic of tests/dcgan_wgp_oracle.py with src/dra_gan.py:59's sigmoid output, and its D gradient two
ways:
  * autograd_d_step: src/dra_gan.py:186-221 literally (torch.autograd.grad with create_graph=True, then backward);
  * closed_form_d_step: what gm_b200.DcganEngine(variant="dra") runs (DESIGN.md §6b) - the NS rows on real / fake, and for
    x_hat the beta chain seeded with 1 (J = ds/dx_hat), ||g|| = sigma' ||J||, the tangent seed
    r = k sigma' [J/||J|| + (1 - 2 sigma) ||J|| x_hat] with k = 2 lam inv (||g|| - K), the tangent pass under x_hat's
    LeakyReLU masks and one weight gradient per layer, shared with the WGAN-GP oracle.  q = bf16_points rounds every tensor
    the device stores in bf16 at the same places.
"""
import torch
import torch.nn.functional as F

import dcgan_wgp_oracle as W
from dcgan_wgp_oracle import _betas, _lrelu_grad, _wgrads, _id, bf16_points  # noqa: F401

EPS = 1e-8


class SigmoidCritic(W.Critic):
    def __init__(self, hd=64, ch=3):
        super().__init__(hd, ch, "none")
        self.out_act = "sigmoid"

    def out(self, s):
        return torch.sigmoid(s)


def make_xhat(real, delta, u, C=1.0):
    """src/dra_gan.py:200-205: real [n, ch*4096] flat, delta [n], u like real (NCHW-flattened)"""
    d = delta.reshape(-1, 1).to(real.dtype)
    return d * real + (1 - d) * (real + C * real.std() * u)


def closed_form_d_step(D, real, fake, xh, lam=10.0, K=1.0, inv=None, q=_id):
    """-> dict(loss, ns, gp, grads [5], parts, norms (||g||), J, r, s) for flat images real / fake / xh [n, ch*4096]; inv scales
    the gradients (1 / global batch), the losses are means over the n images"""
    n = real.shape[0]
    inv = 1.0 / n if inv is None else inv
    with torch.no_grad():
        parts = {}
        ns = 0.0
        for x, key in ((real, "real"), (fake, "fake")):
            s, acts = D.trace(x, q)
            d = torch.sigmoid(s)
            if key == "real":
                ns = ns - torch.log(d + EPS).mean()
                seed = -inv * d * (1 - d) / (d + EPS)
            else:
                ns = ns - torch.log(1 - d + EPS).mean()
                seed = inv * d * (1 - d) / (1 - d + EPS)
            betas, _ = _betas(D, acts, q(seed), q)
            parts[key] = _wgrads(D, acts, betas)
        s, acts = D.trace(xh, q)
        betas, J = _betas(D, acts, torch.ones_like(s), q)
        nJ = J.reshape(n, -1).norm(dim=1)
        sg = torch.sigmoid(s)
        sp = sg * (1 - sg)
        norms = sp * nJ
        k = 2 * lam * inv * (norms - K) * sp
        live = (nJ > 0).view(n, 1, 1, 1)
        xq = q(xh).view(J.shape)
        r = torch.where(live, k.view(n, 1, 1, 1) * (J / nJ.clamp_min(1e-300).view(n, 1, 1, 1)
                                                      + ((1 - 2 * sg) * nJ).view(n, 1, 1, 1) * xq), torch.zeros_like(J))
        r = q(r)
        gp = lam * ((norms - K) ** 2).mean()
        ws = [q(l.weight) for l in D.layers()]
        t = [r]
        for l in range(4):
            t.append(q(_lrelu_grad(acts[l + 1]) * q(F.conv2d(t[-1], ws[l], None, 2, 1))))
        parts["penalty"] = _wgrads(D, t, betas)
        grads = [a + b + c for a, b, c in zip(parts["real"], parts["fake"], parts["penalty"])]
    return dict(loss=ns + gp, ns=ns, gp=gp, grads=grads, parts=parts, norms=norms, J=J, r=r, s=s)


def autograd_d_step(D, real, fake, xh, lam=10.0, K=1.0):
    """src/dra_gan.py:186-221 with this critic: D_loss and its gradient w.r.t. every weight"""
    DX, DG = D(real), D(fake)
    ns = -torch.mean(torch.log(DX + EPS) + torch.log(1 - DG + EPS))
    xh = xh.detach().clone().requires_grad_(True)
    Di = D(xh)
    g = torch.autograd.grad(Di, xh, torch.ones_like(Di), create_graph=True, retain_graph=True, only_inputs=True)[0]
    gp = lam * torch.mean((g.norm(2, dim=1) - K) ** 2)
    loss = ns + gp
    grads = torch.autograd.grad(loss, [l.weight for l in D.layers()])
    return dict(loss=loss.detach(), ns=ns.detach(), gp=gp.detach(), grads=[t.detach() for t in grads], norms=g.detach().norm(2, dim=1))
