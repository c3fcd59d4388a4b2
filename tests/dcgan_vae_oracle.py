"""The VAE on the DCGAN conv path — TEST INFRASTRUCTURE, not product code: the plain-PyTorch statement of
DcganEngine(variant="vae") and of the reference's losses (src/vae.py:94-106,193-212), built on oracle/dcgan_torch.py's pieces
(the DCGAN Generator and Discriminator trunk, bf16_points).

  * Encoder: the DCGAN D trunk (BatchNorm on conv 2-4) with the linear heads mu and log_var stacked as one bias-free
    Conv2d(8h, 2z, 4, 1, 0); heads() is its output [n, 2z] (mu, then log_var), as the device's fp32 head rows hold it.
  * Decoder: the DCGAN generator; pre() is its output before the sigmoid.
  * compute_batch: the reference's expression literally, recon = sum (x - out)^2, KL = sum 0.5 (mu^2 + e^lv - lv - 1),
    z = mu + eps e^(lv/2).
  * dpre / dlatent: the closed forms the device runs (gm_sse_sigmoid_rows, vae_dlatent_kernel)."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import dcgan_torch as O


class Encoder(O.Discriminator):
    def __init__(self, hd=64, z=100, ch=3):
        super().__init__(hd, ch)
        self.z = z
        self.l5 = nn.Conv2d(8 * hd, 2 * z, 4, 1, 0, bias=False)

    def heads(self, x):
        return self.logits(x).view(x.shape[0], 2 * self.z)

    def forward(self, x):
        h = self.heads(x)
        return h[:, :self.z], h[:, self.z:]


class Decoder(O.Generator):
    def pre(self, z):
        """the generator's output before the sigmoid, NCHW"""
        q = self.q
        x = q(z).view(z.shape[0], -1, 1, 1)
        x = q(torch.relu(self.bn1(q(F.conv_transpose2d(x, q(self.l1.weight), None, 1, 0)))))
        x = q(torch.relu(self.bn2(q(O.conv_transpose_k4s2(x, q(self.l2.weight), q)))))
        x = q(torch.relu(self.bn3(q(O.conv_transpose_k4s2(x, q(self.l3.weight), q)))))
        x = q(torch.relu(self.bn4(q(O.conv_transpose_k4s2(x, q(self.l4.weight), q)))))
        return O.conv_transpose_k4s2(x, q(self.l5.weight), q)


def load_from_engine_weights(E, G, sd):
    """sd: DcganEngine(variant="vae").torch_weights() (D = the encoder, G = the decoder)"""
    O.load_from_engine_weights(G, E, sd)


def reparameterize(mu, lv, eps):
    return mu + eps * torch.exp(lv / 2)                                               # src/vae.py:105


def kl_divergence(mu, lv):
    return torch.sum(0.5 * (mu ** 2 + torch.exp(lv) - lv - 1))                       # src/vae.py:212


def compute_batch(E, G, x, eps):
    """src/vae.py:193-208 for flat images x [n, ch*4096] and the reparameterisation noise eps [n, z]"""
    mu, lv = E(x)
    out = G(reparameterize(mu, lv, eps))
    return torch.sum((x - out) ** 2), kl_divergence(mu, lv)


def dpre(out, x, scale=1.0):
    """d(scale sum (x - out)^2) / d(pre-sigmoid output) for out = sigmoid(pre)"""
    return 2 * scale * (out - x) * out * (1 - out)


def dlatent(mu, lv, eps, dz, scale=1.0):
    """(dmu, dlv) of recon + KL given dz = d recon / dz: the KL terms plus the reparameterisation's chain"""
    return scale * (mu + dz), scale * (0.5 * (torch.exp(lv) - 1) + 0.5 * dz * eps * torch.exp(lv / 2))
