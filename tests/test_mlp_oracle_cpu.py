"""The VAE oracle's bf16-point hook (oracle.ref_math.vae_step(q=...)): the default stays the exact restatement of the
reference, and the hook acts at the storage points it names."""
import numpy as np

from inputs import VAE_SHAPES, gm_init_weights, images_from_bits, load_case, params_dict, unpack_draws, check_summary
from oracle import ref_math as R


def _case():
    fx = load_case("vae")
    P = params_dict(gm_init_weights(VAE_SHAPES, 4321), np.float64)
    x = images_from_bits(fx).astype(np.float64)
    eps = unpack_draws(fx, "step1_")[0].astype(np.float64)
    return fx, P, x, eps


def test_default_is_exact_and_matches_the_reference():
    fx, P, x, eps = _case()
    recon, kl, g, _ = R.vae_step(P, x, eps)
    recon_i, kl_i, g_i, _ = R.vae_step(P, x, eps, q=lambda name, v: v)
    assert recon == recon_i and kl == kl_i
    for k in g:
        assert np.array_equal(g[k], g_i[k]), k
    assert abs(recon - fx["step1_recon"]) <= 2e-6 * abs(fx["step1_recon"])
    assert abs(kl - fx["step1_kl"]) <= 2e-5 * abs(fx["step1_kl"])
    for k, v in g.items():
        check_summary(fx, "step1_grad_" + k, v, rtol=5e-5)


def test_weight_points_round_the_weights_only():
    """rounding at the "W" points only is the exact step at bf16-rounded weight matrices (biases untouched)"""
    _, P, x, eps = _case()
    only_w = lambda name, v: R.bf16_round(v) if name == "W" else v
    recon, kl, g, _ = R.vae_step(P, x, eps, q=only_w)
    Pq = {k: (R.bf16_round(v) if k.endswith(".weight") else v) for k, v in P.items()}
    recon_r, kl_r, g_r, _ = R.vae_step(Pq, x, eps)
    assert recon == recon_r and kl == kl_r
    for k in g:
        assert np.array_equal(g[k], g_r[k]), k


def test_bf16_points_move_every_gradient_by_bf16_scale():
    _, P, x, eps = _case()
    seen = set()
    recon, kl, g, _ = R.vae_step(P, x, eps)
    recon_q, kl_q, g_q, _ = R.vae_step(P, x, eps, q=lambda name, v: (seen.add(name), R.bf16_points(name, v))[1])
    assert seen == {"W", "x", "h", "z", "da4", "da3", "dml", "da1"}
    assert 0 < abs(recon_q - recon) < 2e-2 * abs(recon) and 0 < abs(kl_q - kl) < 2e-2 * abs(kl)
    for k in g:
        e = np.linalg.norm(g_q[k] - g[k]) / np.linalg.norm(g[k])
        assert 1e-5 < e < 6e-2, (k, e)
