"""InfoGAN on the DCGAN conv path — TEST INFRASTRUCTURE, not product code: the plain-PyTorch statement of the conv Q network
of DcganEngine(variant="info") and of the reference's MI loss (src/info_gan.py:269-304), built on oracle/dcgan_torch.py's
pieces (the DCGAN Generator and Discriminator, bf16_points).

  * QNet: the DCGAN D trunk (BatchNorm on conv 2-4) with a linear Conv2d(8h, nd + nc, 4, 1, 0) head; rows() is the head's
    output [n, nd + nc] (discrete logits, then the continuous code), as the device's fp32 Q rows hold it.
  * mi_loss: train_Q's expression literally, LAMBDA (F.cross_entropy(logits, argmax one-hot) + F.mse_loss(cont, code)) on
    Q(G(noise)), G's output not detached.
  * mi_rows_grad: the upstream gradient gm_info_loss_rows writes, (softmax - onehot) inv lam and 2 (q - c) inv lam / nc."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import dcgan_torch as O


class QNet(O.Discriminator):
    def __init__(self, hd=64, nd=10, nc=10, ch=3):
        super().__init__(hd, ch)
        self.nd, self.nc = nd, nc
        self.l5 = nn.Conv2d(8 * hd, nd + nc, 4, 1, 0, bias=False)

    def rows(self, x):
        return self.logits(x).view(x.shape[0], self.nd + self.nc)

    def forward(self, x):
        r = self.rows(x)
        return r[:, :self.nd], r[:, self.nd:]


def load_from_engine_weights(G, D, Qn, sd):
    """sd: DcganEngine(variant="info").torch_weights()"""
    O.load_from_engine_weights(G, D, sd)
    with torch.no_grad():
        for name, p in Qn.named_parameters():
            p.copy_(sd["Q." + name].to(p.dtype))


def mi_terms(disc, cont, noise, z):
    """(cross entropy, MSE) of src/info_gan.py:294-299 for Q's outputs and the noise [n, z + nd + nc] that made them"""
    nd = disc.shape[1]
    disc_loss = F.cross_entropy(disc, torch.max(noise[:, z:z + nd], 1)[1])
    cont_loss = F.mse_loss(cont, noise[:, z + nd:])
    return disc_loss, cont_loss


def mi_loss(G, Qn, noise, z, lam=1.0):
    """src/info_gan.py:283-304: MI_loss = LAMBDA (disc_loss + cont_loss) on Q(G(noise))"""
    disc, cont = Qn(G(noise))
    d, c = mi_terms(disc, cont, noise, z)
    return lam * (d + c)


def mi_rows_grad(rows, noise, z, nd, nc, inv, lam=1.0):
    """dMI_loss/d(Q's rows) as the device computes it: softmax(logits) - onehot and 2 (q - c) / nc, times inv lam"""
    tgt = noise[:, z:z + nd].argmax(1)
    gd = torch.softmax(rows[:, :nd], 1) - F.one_hot(tgt, nd).to(rows.dtype)
    gc = 2.0 * (rows[:, nd:nd + nc] - noise[:, z + nd:z + nd + nc]) / nc
    return torch.cat([gd, gc], 1) * (inv * lam)
