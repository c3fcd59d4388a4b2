"""Two-grid K-major GEMMs of the train steps (GPU): a main grid of 4-CTA clusters and a 2-CTA companion grid on the SMs it
leaves free (engine.cu launch_pp208) compute exactly what one grid computes.

The companion overlaps the main grid through programmatic dependent launch, so a context with it turned off
(gm_ctx_set_pdl) runs every plan as one grid.  Each case runs one train step of an engine at a ragged batch whose K-major
208-wide plans take the split (B = 128 * 510 + 77: 511 m-tiles with a 77-row last tile; D's first layer over 2B rows:
1022 m-tiles, the last one's second 64-row half skipped), once with the split and once as single grids, and asserts that
losses and updated parameters agree bit for bit and that the split added launches.  Between them the NSGAN, WGAN-GP,
BEGAN and VAE steps reach every fixed epilogue signature of the ping-pong instances: bias + ReLU / sigmoid, the row-dots
DOT_W, DOT_W_MASK, DOT_W_PRE and DOT_SQ, AUX_SIGMOID_GRAD, AUX_RELU_MASK, AUX_NONZERO_MASK, AUX_L1 and AUX_VAE_OUT; the
single grids themselves are checked element by element against float64 in test_gemm_pingpong4_gpu.py and the engine
tests."""
import pytest
import torch

from mlp_harness import gan_engine

pytestmark = pytest.mark.gpu

B = 128 * 510 + 77


def _set_pdl(eng, on):
    from gm_b200 import _lib
    _lib.check(eng.h, _lib.lib().gm_ctx_set_pdl(eng.h, 1 if on else 0))


def _inputs(x_dim=784, z_dim=20):
    g = torch.Generator().manual_seed(7)
    x = (torch.rand(B, x_dim, generator=g) < 0.3).float().cuda()
    z1, z2 = torch.randn(B, z_dim, generator=g).cuda(), torch.randn(B, z_dim, generator=g).cuda()
    return x, z1, z2


def _gan_step(variant, pdl):
    import gm_b200
    eng = gan_engine(variant, max_batch=B)
    _set_pdl(eng, pdl)
    x, z1, z2 = _inputs()
    hp = gm_b200.AdamHP.make(2e-4)
    torch.cuda.synchronize()
    n0 = gm_b200.launch_count()
    ld = eng.d_grad(x, noise=z1, seed=3).clone()
    eng.apply(1, hp)
    lg = eng.g_grad(B, noise=z2, seed=3).clone()
    eng.apply(0, hp)
    torch.cuda.synchronize()
    out = [ld, lg, eng.params[0].clone(), eng.params[1].clone()]
    launches = gm_b200.launch_count() - n0
    _set_pdl(eng, True)
    del eng
    return out, launches


def _vae_step(pdl):
    import gm_b200
    eng = gm_b200.VaeEngine(784, 400, 20, max_batch=B)
    g = torch.Generator().manual_seed(11)
    eng.params.copy_(0.05 * torch.randn(eng.params.numel(), generator=g).cuda())
    eng.sync_shadows()
    _set_pdl(eng, pdl)
    x, _, _ = _inputs()
    torch.cuda.synchronize()
    n0 = gm_b200.launch_count()
    loss = eng.grad(x, seed=5).clone()
    eng.apply(gm_b200.AdamHP.make(1e-3))
    torch.cuda.synchronize()
    out = [loss, eng.params.clone()]
    launches = gm_b200.launch_count() - n0
    _set_pdl(eng, True)
    del eng
    return out, launches


def _same_bits(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.shape == v.shape and torch.equal(u.view(torch.int32), v.view(torch.int32)), (what, i)


@pytest.mark.parametrize("variant", ["ns", "wgp", "began"])
def test_gan_step_two_grids_match_one_grid(variant):
    split, n_split = _gan_step(variant, True)
    single, n_single = _gan_step(variant, False)
    assert bool(torch.isfinite(split[0]).all()) and bool(torch.isfinite(split[1]).all())
    _same_bits(split, single, variant)
    assert n_split > n_single, (n_split, n_single)


def test_vae_step_two_grids_match_one_grid():
    split, n_split = _vae_step(True)
    single, n_single = _vae_step(False)
    assert bool(torch.isfinite(split[0]).all())
    _same_bits(split, single, "vae")
    assert n_split > n_single, (n_split, n_single)
