"""DCGAN oracle — TEST INFRASTRUCTURE, not product code.

The reference has no convolutional model (README.md:68 recommends DCGAN, README.md:96 lists it as To-Do), so parity for
BASELINE configs[4] is "doubly unpinned" (SURVEY.md 8f): this file is OUR plain-PyTorch fp32 statement of the
architecture (torch.nn Conv2d / ConvTranspose2d / BatchNorm2d on the CPU) driven by the reference's own NSGAN
formulas — train_D: -mean(log(D(x)+1e-8) + log(1-D(G(z))+1e-8)) (src/ns_gan.py:191-192), train_G:
-mean(log(D(G(z))+1e-8)) (src/ns_gan.py:214), D(images) and D(G(z)) as separate forward calls (BatchNorm statistics per
call), autograd backward, torch.optim.Adam.  tests/test_dcgan_gpu.py compares the CUDA conv path with it.

The batch-norm-free Critic of DcganEngine(variant="wgp" / "dra") and its penalised D gradient two ways:
  * autograd_d_step: src/w_gp_gan.py:186-218 / src/dra_gan.py:186-221 literally (torch.autograd.grad with
    create_graph=True, then backward);
  * closed_form_d_step: the steps the CUDA path runs (DESIGN.md §6b) - the loss rows on real / fake, the primal forward at
    x_hat, the input-gradient chain, the per-image tangent seed of the penalty, the tangent forward under x_hat's
    LeakyReLU masks and one conv weight gradient per layer - written with torch.nn.grad's conv2d_input / conv2d_weight.
    With q = bf16_points it rounds every tensor the device stores in bf16 at the same places."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

SLOPE = 0.2
EPS = 1e-8                                                          # the reference's log(D + 1e-8)


def _id(t):
    return t


def bf16_points(t):
    """Rounding model of the CUDA path: every tensor it stores as a bf16 GEMM operand / activation (weights' operand
    copies, z, conv outputs before BatchNorm, activations, the generated image) is rounded to bf16 in the forward pass;
    autograd treats the rounding as identity (the CUDA path applies the bf16-weight gradient to the fp32 master too)."""
    return t + (t.to(torch.bfloat16).to(t.dtype) - t).detach()


def conv_transpose_k4s2(x, w, q=_id):
    """ConvTranspose2d(k=4, s=2, p=1) written the way the CUDA path computes it: one matrix product per input pixel
    (col = x Wm^T, [(kh, kw, co)] columns) followed by the fold of the tap columns (col2im).  With q = identity this is
    F.conv_transpose2d; with q = bf16_points the tap columns are rounded to bf16 before they are summed, as on the device."""
    B, Cin, H, W = x.shape
    Cout = w.shape[1]
    xr = x.permute(0, 2, 3, 1).reshape(B * H * W, Cin)
    Wm = w.permute(2, 3, 1, 0).reshape(16 * Cout, Cin)
    col = q(xr @ Wm.t())
    cols = col.view(B, H * W, 16, Cout).permute(0, 3, 2, 1).reshape(B, Cout * 16, H * W)
    return F.fold(cols, (2 * H, 2 * W), 4, padding=1, stride=2)


class Generator(nn.Module):
    q = staticmethod(_id)          # set to bf16_points to model the CUDA path's storage rounding

    def __init__(self, hd=64, z=100, ch=3):
        super().__init__()
        c = [8 * hd, 4 * hd, 2 * hd, hd, ch]
        self.l1 = nn.ConvTranspose2d(z, c[0], 4, 1, 0, bias=False)
        self.l2 = nn.ConvTranspose2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.ConvTranspose2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.ConvTranspose2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.ConvTranspose2d(c[3], c[4], 4, 2, 1, bias=False)
        self.bn1, self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[:4])

    def forward(self, z):
        q = self.q
        x = q(z).view(z.shape[0], -1, 1, 1)
        x = q(torch.relu(self.bn1(q(F.conv_transpose2d(x, q(self.l1.weight), None, 1, 0)))))
        x = q(torch.relu(self.bn2(q(conv_transpose_k4s2(x, q(self.l2.weight), q)))))
        x = q(torch.relu(self.bn3(q(conv_transpose_k4s2(x, q(self.l3.weight), q)))))
        x = q(torch.relu(self.bn4(q(conv_transpose_k4s2(x, q(self.l4.weight), q)))))
        x = q(torch.sigmoid(conv_transpose_k4s2(x, q(self.l5.weight), q)))
        return x.reshape(z.shape[0], -1)                                    # flat [B, ch*64*64] like src/ns_gan.py:46


class Discriminator(nn.Module):
    q = staticmethod(_id)

    def __init__(self, hd=64, ch=3):
        super().__init__()
        c = [hd, 2 * hd, 4 * hd, 8 * hd]
        self.ch = ch
        self.l1 = nn.Conv2d(ch, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], 1, 4, 1, 0, bias=False)
        self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])

    def logits(self, x):
        q = self.q
        x = q(x).view(x.shape[0], self.ch, 64, 64)                         # un-flatten (src/ns_gan.py:225 flattens)
        x = q(F.leaky_relu(F.conv2d(x, q(self.l1.weight), None, 2, 1), 0.2))
        x = q(F.leaky_relu(self.bn2(q(F.conv2d(x, q(self.l2.weight), None, 2, 1))), 0.2))
        x = q(F.leaky_relu(self.bn3(q(F.conv2d(x, q(self.l3.weight), None, 2, 1))), 0.2))
        x = q(F.leaky_relu(self.bn4(q(F.conv2d(x, q(self.l4.weight), None, 2, 1))), 0.2))
        return F.conv2d(x, q(self.l5.weight), None, 1, 0).view(-1, 1)

    def forward(self, x):
        return torch.sigmoid(self.logits(x))


def load_from_engine_weights(G, D, sd):
    """sd: DcganEngine.torch_weights()."""
    with torch.no_grad():
        for tag, net in (("G", G), ("D", D)):
            for name, p in net.named_parameters():
                p.copy_(sd["%s.%s" % (tag, name)].to(p.dtype))


def d_loss(G, D, images, z):
    return -torch.mean(torch.log(D(images) + 1e-8) + torch.log(1 - D(G(z)) + 1e-8))      # src/ns_gan.py:191-192


def g_loss(G, D, z):
    return -torch.mean(torch.log(D(G(z)) + 1e-8))                                          # src/ns_gan.py:214


class Critic(nn.Module):
    """Conv(ch, h, 4, 2, 1) LReLU -> Conv(h, 2h) LReLU -> Conv(2h, 4h) LReLU -> Conv(4h, 8h) LReLU -> Conv(8h, 1, 4, 1, 0)
    -> relu (out_act="relu", src/w_gp_gan.py:61), identity ("none") or sigmoid ("sigmoid", src/dra_gan.py:59).  No
    BatchNorm, no biases."""

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
        if self.out_act == "sigmoid":
            return torch.sigmoid(s)
        return torch.relu(s) if self.out_act == "relu" else s

    def forward(self, x):
        return self.out(self.trace(x)[0]).view(-1, 1)


def interpolate(real, fake, eps, q=_id):
    """WGAN-GP's x_hat = eps x + (1 - eps) G(z), one eps per image (src/w_gp_gan.py:197-199)"""
    e = eps.view(real.shape[0], 1).to(real.dtype)
    return q(e * q(real) + (1 - e) * q(fake))


def make_xhat(real, delta, u, C=1.0):
    """DRAGAN's x_hat (src/dra_gan.py:200-205): real [n, ch*4096] flat, delta [n], u like real (NCHW-flattened)"""
    d = delta.reshape(-1, 1).to(real.dtype)
    return d * real + (1 - d) * (real + C * real.std() * u)


def _lrelu_grad(y):
    return torch.where(y > 0, torch.ones_like(y), torch.full_like(y, SLOPE))


def _seed(D, s):
    """the x_hat rows' seed of the input-gradient chain: out'(s) for relu (1[s > 0]) and none, 1 for the sigmoid critic,
    whose sigma' enters through the penalty coefficient"""
    return (s > 0).to(s.dtype) if D.out_act == "relu" else torch.ones_like(s)


def _betas(D, acts, seed, q=_id):
    """input-gradient chain: [beta_1, .., beta_5] (pre-activation gradients, beta_5 = seed) and the image gradient.
    The gradient through a k4 s2 p1 conv is the transposed conv written as the device runs it (one product per pixel into
    16 tap columns, then the fold, conv_transpose_k4s2), so that q also rounds the tap columns."""
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


def _rows(D, s, real, inv):
    """the loss rows of real (real=True) or fake logits s and their upstream gradient dL/ds: WGAN-GP's W rows
    (mean(D(G(z))) - mean(D(x))) for the relu / linear critic, the NS rows for the sigmoid one"""
    if D.out_act != "sigmoid":
        sign = -1.0 if real else 1.0
        return sign * D.out(s).mean(), sign * inv * _seed(D, s)
    d = torch.sigmoid(s)
    if real:
        return -torch.log(d + EPS).mean(), -inv * d * (1 - d) / (d + EPS)
    return -torch.log(1 - d + EPS).mean(), inv * d * (1 - d) / (1 - d + EPS)


def _penalty_seed(D, J, s, xh, lam, K, inv, q):
    """(||g|| per image, tangent seed r = d(penalty)/d(x_hat's input gradient)) from J = the chain's image gradient at
    x_hat.  WGAN-GP: g = J, r = 2 lam inv (||g|| - K) g / ||g||.  DRAGAN: g = sigma' J, and since sigma' depends on x_hat too,
    r = k sigma' [J/||J|| + (1 - 2 sigma) ||J|| x_hat] with k = 2 lam inv (||g|| - K).  r = 0 where the gradient is 0."""
    n = s.shape[0]
    if D.out_act != "sigmoid":
        norms = J.reshape(n, -1).norm(dim=1)
        coef = torch.where(norms > 0, 2 * lam * inv * (norms - K) / norms.clamp_min(1e-30), torch.zeros_like(norms))
        return norms, q(coef.view(n, 1, 1, 1) * J)
    nJ = J.reshape(n, -1).norm(dim=1)
    sg = torch.sigmoid(s)
    sp = sg * (1 - sg)
    norms = sp * nJ
    k = 2 * lam * inv * (norms - K) * sp
    live = (nJ > 0).view(n, 1, 1, 1)
    xq = q(xh).view(J.shape)
    r = torch.where(live, k.view(n, 1, 1, 1) * (J / nJ.clamp_min(1e-300).view(n, 1, 1, 1)
                                                  + ((1 - 2 * sg) * nJ).view(n, 1, 1, 1) * xq), torch.zeros_like(J))
    return norms, q(r)


def closed_form_d_step(D, real, fake, xh, lam=10.0, K=1.0, inv=None, q=_id):
    """-> dict(loss, rows, gp, grads [5 weight tensors], parts, norms (||g||), J, r (tangent seed, NCHW), s (x_hat logits))
    for flat images real / fake / xh [n, ch*4096]; inv scales the gradients (1 / global batch), the losses are means over
    the n images"""
    n = real.shape[0]
    inv = 1.0 / n if inv is None else inv
    with torch.no_grad():
        parts = {}
        rows = 0.0
        for x, key in ((real, "real"), (fake, "fake")):
            s, acts = D.trace(x, q)
            loss, seed = _rows(D, s, key == "real", inv)
            rows = rows + loss
            betas, _ = _betas(D, acts, q(seed), q)
            parts[key] = _wgrads(D, acts, betas)
        # penalty: 1. primal forward at x_hat, 2. chain to the image, 3. per-image norm and tangent seed
        s, acts = D.trace(xh, q)
        betas, J = _betas(D, acts, _seed(D, s), q)
        norms, r = _penalty_seed(D, J, s, xh, lam, K, inv, q)
        gp = lam * ((norms - K) ** 2).mean()
        # 4. tangent forward under x_hat's masks, 5. one weight gradient per layer
        ws = [q(l.weight) for l in D.layers()]
        t = [r]
        for l in range(4):
            t.append(q(_lrelu_grad(acts[l + 1]) * q(F.conv2d(t[-1], ws[l], None, 2, 1))))
        parts["penalty"] = _wgrads(D, t, betas)
        grads = [a + b + c for a, b, c in zip(parts["real"], parts["fake"], parts["penalty"])]
    return dict(loss=rows + gp, rows=rows, gp=gp, grads=grads, parts=parts, norms=norms, J=J, r=r, s=s)


def autograd_d_step(D, real, fake, xh, lam=10.0, K=1.0):
    """src/w_gp_gan.py:186-218 (relu / linear critic) or src/dra_gan.py:186-221 (sigmoid) with this critic: D_loss and its
    gradient w.r.t. every critic weight"""
    DX, DG = D(real), D(fake)
    if D.out_act == "sigmoid":
        rows = -torch.mean(torch.log(DX + EPS) + torch.log(1 - DG + EPS))
    else:
        rows = torch.mean(DG) - torch.mean(DX)
    xh = xh.detach().clone().requires_grad_(True)
    Di = D(xh)
    g = torch.autograd.grad(Di, xh, torch.ones_like(Di), create_graph=True, retain_graph=True, only_inputs=True)[0]
    gp = lam * torch.mean((g.norm(2, dim=1) - K) ** 2)
    loss = rows + gp
    grads = torch.autograd.grad(loss, [l.weight for l in D.layers()])
    return dict(loss=loss.detach(), rows=rows.detach(), gp=gp.detach(), grads=[t.detach() for t in grads],
                norms=g.detach().norm(2, dim=1))
