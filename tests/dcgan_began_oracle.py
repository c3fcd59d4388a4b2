"""BEGAN on the DCGAN conv path — TEST INFRASTRUCTURE, not product code: the plain-PyTorch statement of the conv
autoencoder D of DcganEngine(variant="be") and of the reference's BEGAN losses (src/be_gan.py:225-256), built on
oracle/dcgan_torch.py's pieces (bf16_points, the device-shaped transposed convolution, the DCGAN Generator).

  * AutoEncoder: encoder = the DCGAN D trunk ending in a linear Conv2d(8h, e, 4, 1, 0); decoder = the generator stack with
    e in place of z and a linear output.  With q = bf16_points it rounds every tensor the device stores in bf16 in the
    forward pass, with gq = bf16_grad_points every gradient the device stores in bf16 in the backward pass.
  * d_loss / g_loss: the reference's formulas; `signs` lets the L1 terms take given signs as their gradient (the device's,
    where its bf16 reconstruction and the oracle's fall on different sides of the target) while the value stays |r - x|.
  * g_input_grad: the decomposition the device runs for the G step, dL/dG(z) = T - sign(r - G(z)) inv, with T the
    autoencoder's input-gradient chain written with torch.nn.grad's conv-input functions and BatchNorm's training-mode
    backward by hand."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.grad import conv2d_input

from oracle import dcgan_torch as O

SLOPE = 0.2


class _RoundGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


def bf16_grad_points(t):
    """identity in the forward pass; rounds the gradient w.r.t. t to bf16 in the backward pass (where the CUDA path stores
    that gradient as bf16: dL/dr, the BatchNorm backward outputs, the GEMM input gradients, the embedding gradient)"""
    return _RoundGrad.apply(t)


class AutoEncoder(nn.Module):
    q = staticmethod(O._id)
    gq = staticmethod(O._id)

    def __init__(self, hd=64, e=100, ch=3):
        super().__init__()
        self.ch = ch
        c, g = [hd, 2 * hd, 4 * hd, 8 * hd], [8 * hd, 4 * hd, 2 * hd, hd, ch]
        self.encoder, self.decoder = nn.Module(), nn.Module()
        enc, dec = self.encoder, self.decoder
        enc.l1 = nn.Conv2d(ch, c[0], 4, 2, 1, bias=False)
        enc.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        enc.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        enc.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        enc.l5 = nn.Conv2d(c[3], e, 4, 1, 0, bias=False)
        enc.bn2, enc.bn3, enc.bn4 = (nn.BatchNorm2d(k) for k in c[1:])
        dec.l1 = nn.ConvTranspose2d(e, g[0], 4, 1, 0, bias=False)
        dec.l2 = nn.ConvTranspose2d(g[0], g[1], 4, 2, 1, bias=False)
        dec.l3 = nn.ConvTranspose2d(g[1], g[2], 4, 2, 1, bias=False)
        dec.l4 = nn.ConvTranspose2d(g[2], g[3], 4, 2, 1, bias=False)
        dec.l5 = nn.ConvTranspose2d(g[3], g[4], 4, 2, 1, bias=False)
        dec.bn1, dec.bn2, dec.bn3, dec.bn4 = (nn.BatchNorm2d(k) for k in g[:4])

    def trace(self, x):
        """flat [n, ch*4096] -> (reconstruction flat, saved tensors of every layer for g_input_grad)"""
        q, gq, enc, dec = self.q, self.gq, self.encoder, self.decoder
        n = x.shape[0]
        x = gq(q(x).view(n, self.ch, 64, 64))                                         # T, the image gradient
        sv = {"x": x}
        y = q(F.leaky_relu(gq(F.conv2d(x, q(enc.l1.weight), None, 2, 1)), SLOPE))     # dL/d(conv 1), LReLU' applied
        sv["y1"] = y
        for i in (2, 3, 4):
            c = gq(q(F.conv2d(y, q(getattr(enc, "l%d" % i).weight), None, 2, 1)))     # BatchNorm backward output
            y = gq(q(F.leaky_relu(getattr(enc, "bn%d" % i)(c), SLOPE)))               # the GEMM / col2im input gradient
            sv["ec%d" % i], sv["y%d" % i] = c, y
        h = gq(q(F.conv2d(y, q(enc.l5.weight), None, 1, 0)))                         # the linear embedding [n, e, 1, 1]
        sv["h"] = h
        c = gq(q(F.conv_transpose2d(h, q(dec.l1.weight), None, 1, 0)))
        for i in (1, 2, 3, 4):
            a = gq(q(torch.relu(getattr(dec, "bn%d" % i)(c))))
            sv["dc%d" % i], sv["a%d" % i] = c, a
            c = gq(q(O.conv_transpose_k4s2(a, q(getattr(dec, "l%d" % (i + 1)).weight), q)))   # last: dL/dr
        return c.reshape(n, -1), sv                                                   # linear output (src/be_gan.py:73-76)

    def forward(self, x):
        return self.trace(x)[0]


def load_from_engine_weights(G, AE, sd):
    """sd: DcganEngine(variant="be").torch_weights()"""
    O.load_from_engine_weights(G, AE, sd)


def l1(r, x, s=None):
    """per-image sum |r - x|; with s (detached, +-1 / 0) its gradient w.r.t. r - x is s"""
    d = r - x
    if s is None:
        return d.abs().sum(1)
    return ((d.abs() - s * d).detach() + s * d).sum(1)


def d_loss(AE, images, fake, K, signs=(None, None)):
    """src/be_gan.py:224-236 on given images and G(z) (both flat, as D reads them): (D_loss, DX, DG)"""
    DX = l1(AE(images), images, signs[0]).mean()
    DG = l1(AE(fake), fake, signs[1]).mean()
    return DX - K * DG, DX, DG


def g_loss(AE, G, z, sign=None):
    """src/be_gan.py:251-256: G_output is not detached, so the gradient reaches it through D and through the target"""
    fake = G(z)
    return l1(AE(fake), fake, sign).mean()


def _bn_backward(dy, c, bn):
    """BatchNorm2d's training-mode backward (batch statistics, biased variance) of dy w.r.t. its input c"""
    dims = (0, 2, 3)
    N = c.numel() // c.shape[1]
    mu = c.mean(dims, keepdim=True)
    invstd = (c.var(dims, unbiased=False, keepdim=True) + bn.eps).rsqrt()
    xh = (c - mu) * invstd
    dxh = dy * bn.weight.view(1, -1, 1, 1)
    return invstd / N * (N * dxh - dxh.sum(dims, keepdim=True) - xh * (dxh * xh).sum(dims, keepdim=True))


def g_input_grad(AE, fake, inv):
    """dL/dG(z) of the G loss inv sum_i |AE(f_i) - f_i| the way the device composes it: dr = sign(r - f) inv, the decoder's and
    encoder's input-gradient chain of dr (no weight gradients) gives T, and dL/df = T - dr.  fake flat [n, ch*4096]."""
    enc, dec = AE.encoder, AE.decoder
    with torch.no_grad():
        r, sv = AE.trace(fake)
        n = fake.shape[0]
        dr = (torch.sign(r - fake) * inv).view(n, AE.ch, 64, 64)
        d = dr
        for i in (4, 3, 2, 1):                                           # decoder: convT_{i+1} input, then ReLU, BatchNorm i
            d = F.conv2d(d, getattr(dec, "l%d" % (i + 1)).weight, None, 2, 1)
            d = _bn_backward(d * (sv["a%d" % i] > 0).to(d.dtype), sv["dc%d" % i], getattr(dec, "bn%d" % i))
        d = F.conv2d(d, dec.l1.weight, None, 1, 0)                        # dL/d(embedding) [n, e, 1, 1]
        d = conv2d_input(sv["y4"].shape, enc.l5.weight, d, 1, 0)
        for i in (4, 3, 2):                                              # encoder: LeakyReLU', BatchNorm i, conv_i input
            d = d * O._lrelu_grad(sv["y%d" % i])
            d = _bn_backward(d, sv["ec%d" % i], getattr(enc, "bn%d" % i))
            d = conv2d_input(sv["y%d" % (i - 1)].shape, getattr(enc, "l%d" % i).weight, d, 2, 1)
        d = d * O._lrelu_grad(sv["y1"])
        T = conv2d_input(sv["x"].shape, enc.l1.weight, d, 2, 1)
        return (T - dr).reshape(n, -1)
