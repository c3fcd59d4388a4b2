"""The autoencoder on the DCGAN conv path — TEST INFRASTRUCTURE, not product code: the plain-PyTorch statement of
DcganEngine(variant="ae") and of the reference's loss (src/ae.py:38-39,147-160), built on oracle/dcgan_torch.py's pieces.

  * Encoder: the DCGAN D trunk (BatchNorm on conv 2-4) with a bias-free linear head Conv2d(8h, z, 4, 1, 0); head() is its
    output h [n, z] (the device's fp32 head rows), forward() the code relu(h).
  * Decoder: the DCGAN generator with pre(), its output before the sigmoid (tests/dcgan_vae_oracle.py).
  * compute_batch: the reference's expression literally, sum (x - decoder(encoder(x)))^2.
  * step: the decomposition the device runs - encoder forward, relu code, decoder forward, the SSE's dL/d(pre-sigmoid)
    (gm_sse_sigmoid_rows), dz through the decoder, dh = dz 1[h > 0] (gm_ae_dlatent_rows), the encoder backward."""
import torch
import torch.nn as nn

from oracle import dcgan_torch as O
from dcgan_vae_oracle import Decoder, dpre  # noqa: F401


class Encoder(O.Discriminator):
    def __init__(self, hd=64, z=32, ch=3):
        super().__init__(hd, ch)
        self.z = z
        self.l5 = nn.Conv2d(8 * hd, z, 4, 1, 0, bias=False)

    def head(self, x):
        return self.logits(x).view(x.shape[0], self.z)

    def forward(self, x):
        return torch.relu(self.head(x))


def load_from_engine_weights(E, G, sd):
    """sd: DcganEngine(variant="ae").torch_weights() (D = the encoder, G = the decoder)"""
    O.load_from_engine_weights(G, E, sd)


def compute_batch(E, G, x):
    """src/ae.py:147-160 for flat images x [n, ch*4096]"""
    return torch.sum((x - G(E(x))) ** 2)


def dlatent(h, dz):
    """dL/dh of the code relu(h) given dz = dL/dcode (0 where h <= 0, as torch's relu backward)"""
    return torch.where(h > 0, dz, torch.zeros_like(dz))


def step(E, G, x):
    """-> dict(loss, h, code, out, dpre, dz, dh, grads: {"D.<name>" / "G.<name>": gradient}) of compute_batch, formed by the
    device's decomposition; autograd runs each network's backward alone, with the upstream the previous stage produced"""
    n = x.shape[0]
    h = E.head(x)
    code = torch.relu(h)
    zc = code.detach().requires_grad_(True)
    pre = G.pre(zc)
    out = torch.sigmoid(pre).reshape(n, -1)
    loss = torch.sum((x - out.detach()) ** 2)
    dp = dpre(out.detach(), x).view(pre.shape)
    gG = torch.autograd.grad(pre, [zc] + list(G.parameters()), dp)
    dz = gG[0]
    dh = dlatent(h.detach(), dz)
    gE = torch.autograd.grad(h, list(E.parameters()), dh)
    grads = {"D." + k: g for (k, _), g in zip(E.named_parameters(), gE)}
    grads.update({"G." + k: g for (k, _), g in zip(G.named_parameters(), gG[1:])})
    return dict(loss=loss.detach(), h=h.detach(), code=code.detach(), out=out.detach(), dpre=dp, dz=dz, dh=dh, grads=grads)
