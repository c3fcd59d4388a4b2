"""The MLP InfoGAN's train_Q (src/info_gan.py:269-304) on the GPU: MI_loss.backward() puts on model.G and model.Q exactly
the G and Q gradients the fused MI kernels computed in that train_Q call, even after a later call overwrote the engine's
gradient buffers."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _flat(mod):
    return torch.cat([p.grad.reshape(-1) for p in mod.parameters()])


def test_train_q_backward_delivers_the_gradients_of_its_call():
    import info_gan
    from gm_b200.gan_api import G_NET
    torch.manual_seed(0)
    model = info_gan.InfoGAN(784, 400, 20, 10, 10)
    images = (torch.rand(32, 784) < 0.13).float()
    it = [(images.view(32, 1, 28, 28), torch.zeros(32, dtype=torch.long))]
    tr = info_gan.InfoGANTrainer(model, it, it, it)
    first = tr.train_Q(images)
    eng = tr._engine
    want_g, want_q = eng.grads[G_NET].clone(), eng.q_grads.clone()
    second = tr.train_Q(images)                                      # fresh codes: overwrites the engine's gradients
    assert not torch.equal(eng.grads[G_NET], want_g) and not torch.equal(eng.q_grads, want_q)
    first.backward()
    assert torch.equal(_flat(model.G), want_g) and torch.equal(_flat(model.Q), want_q)
    assert all(p.grad is None for p in model.D.parameters())
    for p in model.parameters():
        p.grad = None
    want_g, want_q = eng.grads[G_NET].clone(), eng.q_grads.clone()
    second.backward()
    assert torch.equal(_flat(model.G), want_g) and torch.equal(_flat(model.Q), want_q)
