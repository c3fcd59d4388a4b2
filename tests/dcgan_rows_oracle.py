"""The row losses of the DCGAN conv path's batch-norm D — TEST INFRASTRUCTURE, not product code: every row variant of
oracle/ref_math.py's d_loss / g_loss (mm, w, ls, the six f_*; src/mm_gan.py, src/w_gan.py, src/ls_gan.py, src/f_gan.py)
written in torch on D's sigmoid outputs, with LSGAN's targets a, b, c (src/ls_gan.py:173-215; ref_math fixes 0, 1, 1), so
that autograd through oracle/dcgan_torch.py's G and D gives the reference's gradients."""
import torch

EPS = 1e-8                                                          # the reference's log(D + 1e-8)
F_METHODS = ("total_variation", "forward_kl", "reverse_kl", "pearson", "hellinger", "jensen_shannon")
ROW_VARIANTS = ("mm", "w", "ls") + tuple("f_" + m for m in F_METHODS)


def d_rows(variant, dx, dg, a=0.0, b=1.0):
    """train_D's loss on D(x) = dx and D(G(z)) = dg"""
    m = torch.mean
    if variant in ("ns", "mm"):
        return -m(torch.log(dx + EPS) + torch.log(1 - dg + EPS))
    if variant == "w":
        return m(dg) - m(dx)
    if variant == "ls":
        return 0.5 * m((dx - b) ** 2) + 0.5 * m((dg - a) ** 2)
    f = variant[2:]
    if f == "total_variation":
        return -(m(0.5 * torch.tanh(dx)) - m(0.5 * torch.tanh(dg)))
    if f == "forward_kl":
        return -(m(dx) - m(torch.exp(dg - 1)))
    if f == "reverse_kl":
        return -(m(-torch.exp(dx)) - m(-1 - dg))
    if f == "pearson":
        return -(m(dx) - m(0.25 * dg ** 2 + dg))
    if f == "hellinger":
        return -(m(1 - torch.exp(dx)) - m((1 - torch.exp(dg)) / torch.exp(dg)))
    if f == "jensen_shannon":
        return -(m(2. - (1 + torch.exp(-dx))) - m(-(2. - torch.exp(dg))))
    raise ValueError(variant)


def g_rows(variant, dg, c=1.0):
    """train_G's loss on D(G(z)) = dg"""
    m = torch.mean
    if variant == "ns":
        return -m(torch.log(dg + EPS))
    if variant == "mm":
        return m(torch.log(1 - dg + EPS))
    if variant == "w":
        return -m(dg)
    if variant == "ls":
        return 0.5 * m((dg - c) ** 2)
    f = variant[2:]
    if f == "total_variation":
        return -m(0.5 * torch.tanh(dg))
    if f == "forward_kl":
        return -m(torch.exp(dg - 1))
    if f == "reverse_kl":
        return -m(-1 - dg)
    if f == "pearson":
        return -m(0.25 * dg ** 2 + dg)
    if f == "hellinger":
        return -m((1 - torch.exp(dg)) / torch.exp(dg))
    if f == "jensen_shannon":
        return -m(-(2. - torch.exp(dg)))
    raise ValueError(variant)


def d_loss(G, D, images, z, variant, a=0.0, b=1.0):
    """train_D with D(images) and D(G(z)) as separate calls (BatchNorm statistics per call)"""
    return d_rows(variant, D(images), D(G(z)), a, b)


def g_loss(G, D, z, variant, c=1.0):
    return g_rows(variant, D(G(z)), c)
