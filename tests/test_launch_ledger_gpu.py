"""gm_launch_count is the number of this library's kernels an entry point launched: for a representative call of every
launching path, its delta equals the kernels the CUDA profiler sees (copies, memsets and torch's own at:: kernels left
out) and the launches gm_prof_report counts at level 2."""
import pytest
import torch

from mlp_harness import gan_engine

pytestmark = pytest.mark.gpu

B = 32


def _ledger(fn):
    """(launch-count delta, library kernels in the CUDA trace, launches summed over gm_prof_report) of fn()"""
    import gm_b200
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    gm_b200.prof_report()                     # drops records left by earlier calls
    gm_b200.prof_enable(2)
    try:
        n0 = gm_b200.launch_count()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        delta = gm_b200.launch_count() - n0
        report = sum(n for _, n, _ in gm_b200.prof_report())
    finally:
        gm_b200.prof_enable(0)
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset")) and "at::" not in e.name]
    return delta, kernels, report


def _check(fn):
    delta, kernels, report = _ledger(fn)
    assert delta == len(kernels) == report, (delta, report, kernels)
    assert delta > 0


def _hp():
    import gm_b200
    return gm_b200.AdamHP.make(2e-4)


def _images(n, x=784, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, x, generator=g) < 0.3).float().cuda()


def _noise(n, z, seed=1):
    return torch.randn(n, z, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize("variant", ["ns", "ra", "fisher", "wgp", "dra", "began"])
def test_mlp_gan_step(variant):
    eng = gan_engine(variant, max_batch=64)
    x, z1, z2 = _images(B), _noise(B, 20, 1), _noise(B, 20, 2)
    hp = _hp()
    _check(lambda: eng.d_grad(x, noise=z1))
    _check(lambda: eng.g_grad(B, noise=z2))
    _check(lambda: eng.apply(1, hp))
    _check(lambda: eng.apply(0, hp))


def test_mlp_gan_lazy_gradients():
    eng = gan_engine("ns", max_batch=64)
    x, z = _images(B), _noise(B, 20)
    eng.set_lazy_grads(True)
    eng.d_grad(x, noise=z)
    _check(eng.materialize_grads)
    eng.g_grad(B, noise=z)
    _check(lambda: eng.set_lazy_grads(False))


def test_info_gan_q_step():
    import gm_b200
    eng = gm_b200.InfoGanEngine(784, 400, 20, max_batch=64)
    noise = _noise(B, eng.noise_dim)
    _check(lambda: eng.q_grad(B, noise))
    _check(lambda: eng.apply_mi(_hp()))


def test_custom_path():
    eng = gan_engine("ns", max_batch=64)
    x, z = _images(B), _noise(B, 20)
    _check(lambda: eng.d_forward(0, x))
    dscore = torch.ones(B, device="cuda")
    _check(lambda: eng.d_backward(0, dscore, True))
    _check(lambda: eng.g_forward(z))
    dimg = torch.full((B, 784), 1e-3, device="cuda")
    _check(lambda: eng.g_backward(dimg))


def test_gan_inference_and_debug_entries():
    eng = gan_engine("ns", max_batch=64)
    x, z = _images(B), _noise(B, 20)
    _check(lambda: eng.generate(z))
    _check(lambda: eng.discriminate(x))
    _check(lambda: eng.debug_read("Xall", 0, B, 784))
    _check(lambda: eng.debug_noise(B, 7, 3))
    _check(lambda: eng.sample_indices(B, 5))
    _check(eng.sync_all)


def test_vae():
    import gm_b200
    eng = gm_b200.VaeEngine(784, 400, 20, max_batch=64)
    x, eps = _images(B), _noise(B, 20)
    _check(lambda: eng.grad(x, eps=eps))
    _check(lambda: eng.apply(_hp()))
    _check(lambda: eng.forward(x, eps=eps, want_losses=True))
    _check(lambda: eng.decode(eps))
    _check(lambda: eng.debug_read("H1", 0, B, 400))
    mu, lv = eng.encoder_forward(0, x)
    _check(lambda: eng.encoder_forward(1, x))
    dmu, dlv = torch.full_like(mu, 1e-2), torch.full_like(lv, 1e-2)
    _check(lambda: eng.encoder_backward(1, B, dmu, dlv))
    _check(lambda: eng.decoder_forward(0, eps))
    dimg = torch.full((B, 784), 1e-3, device="cuda")
    _check(lambda: eng.decoder_backward(0, B, dimg, True))


def test_autoencoder():
    import gm_b200
    eng = gm_b200.AeEngine(784, 32, max_batch=64)
    x = _images(B)
    _check(lambda: eng.grad(x))


@pytest.mark.parametrize("out", ["bf16", "fp32_split_k"])
def test_gemm(out):
    import gm_b200
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn(4096, 400, device="cuda", generator=g).to(torch.bfloat16)
    W = torch.randn(208, 400, device="cuda", generator=g).to(torch.bfloat16)
    if out == "bf16":
        C = torch.empty(4096, 208, device="cuda", dtype=torch.bfloat16)
        _check(lambda: gm_b200.gemm_bf16(A, W, C, "nt"))
    else:
        Cf = torch.empty(400, 256, device="cuda")
        Bt = torch.randn(4096, 208, device="cuda", generator=g).to(torch.bfloat16)
        delta, kernels, report = _ledger(lambda: gm_b200.gemm_bf16(A, Bt, Cf, "tn", M=400, N=208, K=4096))
        assert delta == len(kernels) == report == 2, (delta, report, kernels)      # split-K GEMM + reduction


@pytest.mark.parametrize("variant", ["ns", "wgp", "dra", "be", "info", "vae", "ae"])
def test_dcgan_step(variant):
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=16, variant=variant)
    n = 8
    rows = eng.stage_images((torch.rand(n, 3 * 4096, generator=torch.Generator().manual_seed(4)) < 0.3).float().cuda())
    hp = _hp()
    if variant == "vae":
        _check(lambda: eng.vae_grad(rows, n))
        _check(lambda: eng.apply(hp))
        return
    if variant == "ae":
        _check(lambda: eng.ae_grad(rows, n))
        _check(lambda: eng.apply(hp))
        return
    _check(lambda: eng.d_grad(rows, n))
    _check(lambda: eng.g_grad(n))
    _check(lambda: eng.apply(1, hp))
    _check(lambda: eng.apply(0, hp))
    if variant == "info":
        _check(lambda: eng.q_grad(n))
        _check(lambda: eng.apply_mi(hp))
