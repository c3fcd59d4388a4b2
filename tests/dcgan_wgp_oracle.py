"""WGAN-GP conv critic oracle — test infrastructure, not product code.

The batch-norm-free DCGAN critic of gm_b200.DcganEngine(variant="wgp") in plain PyTorch, and its D gradient two ways:
  * autograd_d_step: src/w_gp_gan.py:186-218 literally (torch.autograd.grad with create_graph=True, then backward);
  * closed_form_d_step: the five steps the CUDA path runs (DESIGN.md §6b) - primal forward at x_hat, input-gradient chain
    seeded with 1[s > 0] (or 1), per-image penalty coefficient, tangent forward under the same LeakyReLU masks, and one
    conv weight-gradient per layer - written with torch.nn.grad's conv2d_input / conv2d_weight.  With q = bf16_points it
    rounds every tensor the device stores in bf16 at the same places.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from oracle.dcgan_torch import conv_transpose_k4s2

SLOPE = 0.2


def _id(t):
    return t


def bf16_points(t):
    """round to bf16 in value, identity for autograd (as oracle.dcgan_torch.bf16_points)"""
    return t + (t.to(torch.bfloat16).to(t.dtype) - t).detach()


class Critic(nn.Module):
    """Conv(ch, h, 4, 2, 1) LReLU -> Conv(h, 2h) LReLU -> Conv(2h, 4h) LReLU -> Conv(4h, 8h) LReLU -> Conv(8h, 1, 4, 1, 0)
    -> relu (out_act="relu", src/w_gp_gan.py:61) or identity (out_act="none").  No BatchNorm, no biases."""

    def __init__(self, hd=64, ch=3, out_act="relu"):
        super().__init__()
        c = [hd, 2 * hd, 4 * hd, 8 * hd]
        self.ch, self.out_act = ch, out_act
        self.l1 = nn.Conv2d(ch, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], 1, 4, 1, 0, bias=False)

    def layers(self):
        return [self.l1, self.l2, self.l3, self.l4, self.l5]

    def trace(self, x, q=_id):
        """flat [n, ch*64*64] -> (logits s [n], [x0, y1, .., y4]) with the LeakyReLU outputs y_l (their signs are the masks)"""
        x = q(x.view(x.shape[0], self.ch, 64, 64))
        acts = [x]
        for l in self.layers()[:4]:
            x = q(F.leaky_relu(q(F.conv2d(x, q(l.weight), None, 2, 1)), SLOPE))
            acts.append(x)
        return F.conv2d(x, q(self.l5.weight), None, 1, 0).view(-1), acts

    def out(self, s):
        return torch.relu(s) if self.out_act == "relu" else s

    def forward(self, x):
        return self.out(self.trace(x)[0]).view(-1, 1)


def load_engine_weights(D, sd):
    """sd: DcganEngine.torch_weights() of a wgp engine"""
    with torch.no_grad():
        for name, p in D.named_parameters():
            p.copy_(sd["D." + name].to(p.dtype))


def _lrelu_grad(y):
    return torch.where(y > 0, torch.ones_like(y), torch.full_like(y, SLOPE))


def _seed(D, s):
    return (s > 0).to(s.dtype) if D.out_act == "relu" else torch.ones_like(s)


def _betas(D, acts, seed, q=_id):
    """input-gradient chain: [beta_1, .., beta_5] (pre-activation gradients, beta_5 = seed) and the image gradient.
    The gradient through a k4 s2 p1 conv is the transposed conv written as the device runs it (one product per pixel into
    16 tap columns, then the fold, oracle.dcgan_torch.conv_transpose_k4s2), so that q also rounds the tap columns."""
    ws = [q(l.weight) for l in D.layers()]
    n = seed.shape[0]
    b = seed.view(n, 1, 1, 1)
    betas = [b]
    d = q(conv2d_input(acts[4].shape, ws[4], b, 1, 0))
    for l in range(3, -1, -1):                                       # layer l+1 (0-based l) output acts[l+1]
        b = q(_lrelu_grad(acts[l + 1]) * d)
        betas.insert(0, b)
        d = q(conv_transpose_k4s2(b, ws[l], q))
    return betas, d


def _wgrads(D, inputs, betas):
    shapes = [l.weight.shape for l in D.layers()]
    return [conv2d_weight(inputs[l], shapes[l], betas[l], 2 if l < 4 else 1, 1 if l < 4 else 0) for l in range(5)]


def closed_form_d_step(D, real, fake, eps, lam=10.0, inv=None, q=_id):
    """-> dict(loss, w_part, gp, grads [5 weight tensors], norms, r (tangent seed, NCHW)) for flat images real / fake [n, ch*4096]
    and eps [n]; inv scales the gradients (1 / global batch), the losses are means over the n images"""
    n = real.shape[0]
    inv = 1.0 / n if inv is None else inv
    with torch.no_grad():
        e = eps.view(n, 1).to(real.dtype)
        xh = q(e * q(real) + (1 - e) * q(fake))
        # W part: mean(D(G(z))) - mean(D(x)), dL/ds = +-inv act'(s)
        parts = {}
        w_part = 0.0
        for x, sign, key in ((real, -1.0, "real"), (fake, 1.0, "fake")):
            s, acts = D.trace(x, q)
            w_part = w_part + sign * D.out(s).mean()
            betas, _ = _betas(D, acts, q(sign * inv * _seed(D, s)), q)
            parts[key] = _wgrads(D, acts, betas)
        # penalty: 1. primal forward at x_hat, 2. chain to the image, 3. per-image coefficient
        s, acts = D.trace(xh, q)
        betas, g = _betas(D, acts, _seed(D, s), q)
        norms = g.reshape(n, -1).norm(dim=1)
        coef = torch.where(norms > 0, 2 * lam * inv * (norms - 1) / norms.clamp_min(1e-30), torch.zeros_like(norms))
        r = q(coef.view(n, 1, 1, 1) * g)
        gp = lam * ((norms - 1) ** 2).mean()
        # 4. tangent forward under x_hat's masks, 5. one weight gradient per layer
        ws = [q(l.weight) for l in D.layers()]
        t = [r]
        for l in range(4):
            t.append(q(_lrelu_grad(acts[l + 1]) * q(F.conv2d(t[-1], ws[l], None, 2, 1))))
        parts["penalty"] = _wgrads(D, t, betas)
        grads = [a + b + c for a, b, c in zip(parts["real"], parts["fake"], parts["penalty"])]
    return dict(loss=w_part + gp, w_part=w_part, gp=gp, grads=grads, parts=parts, norms=norms, r=r)


def autograd_d_step(D, real, fake, eps, lam=10.0):
    """src/w_gp_gan.py:186-218 with this critic: D_loss and its gradient w.r.t. every critic weight"""
    n = real.shape[0]
    e = eps.view(n, 1).to(real.dtype).expand(real.shape)
    xh = (e * real + (1 - e) * fake).requires_grad_(True)
    dh = D(xh)
    g = torch.autograd.grad(dh, xh, torch.ones_like(dh), create_graph=True, retain_graph=True, only_inputs=True)[0]
    gp = lam * torch.mean((g.norm(2, dim=1) - 1) ** 2)
    w_part = torch.mean(D(fake)) - torch.mean(D(real))
    loss = w_part + gp
    grads = torch.autograd.grad(loss, [l.weight for l in D.layers()])
    return dict(loss=loss.detach(), w_part=w_part.detach(), gp=gp.detach(), grads=[t.detach() for t in grads],
                norms=g.detach().norm(2, dim=1))
