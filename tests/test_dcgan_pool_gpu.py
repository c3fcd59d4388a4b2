"""The conv path's device-resident 8-bit training set on the GPU: gm_stage_pool_rows against stage_images of the same images,
bit for bit, with the drawn indices against the host twin of the permutation; its keying; its argument checks; and the
trainers with device_dataset on against the same trainers fed the same draws through the host loader path, bitwise."""
import ctypes as C

import pytest
import torch
from torch.utils.data import DataLoader, TensorDataset

from gm_b200 import parallel as par
from gm_b200.dcgan import DevicePool

pytestmark = pytest.mark.gpu
BIG = 1 << 40


def _values(kind, shape, g):
    k = torch.randint(0, 256, shape, generator=g, device="cuda")
    if kind == "binary":
        return (k < 77).float()
    if kind == "k255":
        return k.float() / 255
    if kind == "normalised":
        return (k.float() / 255 - 0.5) / 0.5
    return torch.tensor([0.0, -0.0, 1.0, -1.0, 0.5], device="cuda")[k % 5]


def _pool(images, ch, batch_size=16):
    loader = DataLoader(TensorDataset(images, torch.zeros(images.shape[0])), batch_size=batch_size, shuffle=True)
    pool = DevicePool.from_loader(loader, ch, budget=BIG)
    assert pool is not None and pool.codes.is_cuda
    return pool


def _check_draw(eng, pool, images, rows, seed, round, offset):
    idx = torch.full((rows,), -1, dtype=torch.int32, device="cuda")
    got = eng.stage_pool(pool, rows, seed, round, offset, idx_out=idx)
    want_idx = pool.indices_host(seed, round, offset, rows)
    assert torch.equal(idx.cpu().long(), want_idx)
    want = eng.stage_images(images[want_idx.cuda()].reshape(rows, -1))
    assert got.shape == want.shape and torch.equal(got.view(torch.int16), want.view(torch.int16))
    return idx


@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("kind", ["binary", "k255", "normalised", "signed_zero"])
def test_stage_pool_rows_equal_stage_images(kind, ch):
    import gm_b200
    g = torch.Generator(device="cuda").manual_seed(7 + ch)
    N = 1100                                                          # not a power of two
    images = _values(kind, (N, ch, 64, 64), g)
    pool = _pool(images, ch)
    eng = gm_b200.DcganEngine(hidden_dim=16, z_dim=20, channels=ch)
    for rows, offset in ((1, 0), (1, N - 1), (7, 0), (7, 513), (7, N - 7), (1024, 0), (1024, N - 1024)):
        _check_draw(eng, pool, images, rows, 12345, 3, offset)


def test_a_large_pool_exercises_the_grid_stride_loop():
    import gm_b200
    g = torch.Generator(device="cuda").manual_seed(3)
    N = 20011
    images = _values("k255", (N, 3 * 4096), g)
    pool = _pool(images, 3, batch_size=1024)
    del g
    eng = gm_b200.DcganEngine(hidden_dim=16, z_dim=20)
    idx = _check_draw(eng, pool, images, N, 99, 0, 0)                # every block walks ~19 rows
    assert sorted(idx.cpu().tolist()) == list(range(N))
    _check_draw(eng, pool, images, 5000, 99, 1, N - 5000)


def test_draws_repeat_for_the_same_key_and_differ_otherwise():
    import gm_b200
    g = torch.Generator(device="cuda").manual_seed(4)
    images = _values("k255", (300, 3 * 4096), g)
    pool = _pool(images, 3)
    eng = gm_b200.DcganEngine(hidden_dim=16, z_dim=20)

    def draw(seed, round):
        idx = torch.empty(64, dtype=torch.int32, device="cuda")
        rows = eng.stage_pool(pool, 64, seed, round, idx_out=idx).clone()
        return idx.cpu().tolist(), rows

    base = par.rank_seed(1234, 0) ^ DevicePool.SEED_MIX
    i0, r0 = draw(base, 5)
    i1, r1 = draw(base, 5)
    assert i0 == i1 and torch.equal(r0.view(torch.int16), r1.view(torch.int16))
    assert draw(base, 6)[0] != i0
    assert draw(par.rank_seed(1234, 1) ^ DevicePool.SEED_MIX, 5)[0] != i0
    assert len(set(i0)) == 64


def test_argument_checks_launch_nothing():
    from gm_b200 import _lib
    L, h = _lib.lib(), _lib.ctx()
    codes = torch.zeros(8, 4096, dtype=torch.uint8, device="cuda")
    table = torch.zeros(256, dtype=torch.int16, device="cuda")
    out = torch.zeros(8 * 4096, dtype=torch.bfloat16, device="cuda")
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)                # noqa: E731

    def call(codes_p=None, n_pool=8, row_vals=4096, table_p=None, offset=0, rows=4, out_p=None):
        return L.gm_stage_pool_rows(h, codes_p or p(codes), n_pool, row_vals, table_p or p(table), 1, 2, offset, rows, out_p or p(out),
                                    None, _lib._stream())

    torch.cuda.synchronize()
    _lib.launch_count(reset=True)
    bad = [dict(row_vals=4088), dict(row_vals=0), dict(codes_p=p(codes, 1)), dict(out_p=p(out, 2)), dict(rows=0), dict(rows=-1),
           dict(rows=9), dict(n_pool=0), dict(n_pool=1 << 31, rows=4), dict(offset=5), dict(offset=8, rows=1), dict(offset=1 << 63),
           dict(table_p=p(table, 1))]
    for kw in bad:
        assert call(**kw) == -1, kw                                   # GM_ERR_ARG
    assert L.gm_stage_pool_rows(h, None, 8, 4096, p(table), 1, 2, 0, 4, p(out), None, _lib._stream()) == -1
    assert _lib.launch_count(reset=True) == 0
    assert call(offset=4) == 0 and call(rows=8) == 0
    assert _lib.launch_count(reset=True) == 2


# ------------------------------------------------------------------ the trainers, device_dataset on vs the host path
GANS = {"ns": ("dc_gan", "DCGAN", "DCGANTrainer"), "wgp": ("dc_w_gp_gan", "DCWGPGAN", "DCWGPGANTrainer"),
        "dra": ("dc_dra_gan", "DCDRAGAN", "DCDRAGANTrainer"), "ra": ("dc_ra_gan", "DCRaNSGAN", "DCRaNSGANTrainer"),
        "fisher": ("dc_fisher_gan", "DCFisherGAN", "DCFisherGANTrainer"), "be": ("dc_be_gan", "DCBEGAN", "DCBEGANTrainer"),
        "info": ("dc_info_gan", "DCInfoGAN", "DCInfoGANTrainer")}


def _k255(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, 3, 64, 64), generator=g).float() / 255


def _gan(variant, loader):
    import importlib
    mod, model_cls, tr_cls = GANS[variant]
    M = importlib.import_module(mod)
    torch.manual_seed(3)
    model = getattr(M, model_cls)(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    tr = getattr(M, tr_cls)(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    tr._seed = 4321
    return tr


def _same_training(a, b, lists):
    for name in lists:
        assert getattr(a, name) == getattr(b, name), name
    sa, sb = a.model.state_dict(), b.model.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


@pytest.mark.parametrize("variant", list(GANS))
def test_gan_trainer_with_the_pool_equals_the_host_path_on_the_same_draws(variant):
    images = _k255(64)
    loader = DataLoader(TensorDataset(images, torch.zeros(64)), batch_size=16, shuffle=True)
    a = _gan(variant, loader)
    a.device_dataset = True
    a.train(num_epochs=2, G_lr=2e-4, D_lr=2e-4, D_steps=1)
    assert a._pool is not None
    b = _gan(variant, loader)
    seed = par.rank_seed(b._seed, 0) ^ DevicePool.SEED_MIX
    draws = iter(range(1 << 20))

    def process_batch(iterator):                                        # step * D_steps + k, in the order train() asks
        idx = a._pool.indices_host(seed, next(draws), 0, 16)
        return images[idx].view(16, -1).cuda().contiguous()

    b.process_batch = process_batch
    b.train(num_epochs=2, G_lr=2e-4, D_lr=2e-4, D_steps=1)
    assert len(a.Dlosses) == 8
    _same_training(a, b, ["Dlosses", "Glosses"] + (["MIlosses"] if variant == "info" else []))


def _vae(train_iter, val):
    import dc_vae as M
    torch.manual_seed(5)
    model = M.DCVAE(image_size=64 * 64 * 3, hidden_dim=16, z_dim=20)
    tr = M.DCVAETrainer(model=model, train_iter=train_iter, val_iter=val, test_iter=val, viz=False)
    tr._seed = 777
    return tr


def test_vae_trainer_with_the_pool_equals_the_host_path_on_the_same_epochs():
    N, B = 60, 16                                                      # batches of 16, 16, 16 and 12
    images = _k255(N, 1)
    val = DataLoader(TensorDataset(_k255(16, 2), torch.zeros(16)), batch_size=16, shuffle=False)
    a = _vae(DataLoader(TensorDataset(images, torch.zeros(N)), batch_size=B, shuffle=True), val)
    a.device_dataset = True
    torch.manual_seed(9)                                               # validation draws its eps from torch's stream
    a.train(num_epochs=2)
    seed = par.rank_seed(777, 0) ^ DevicePool.SEED_MIX

    class Epochs:
        """epoch e: the batches of permutation e, as the pool draws them"""
        e = 0

        def __iter__(self):
            perm = a._pool.indices_host(seed, self.e, 0, N)
            self.e += 1
            return iter([(images[perm[k:k + B]], torch.zeros(min(B, N - k))) for k in range(0, N, B)])

    b = _vae(Epochs(), val)
    torch.manual_seed(9)
    b.train(num_epochs=2)
    assert len(a.recon_loss) == 8
    _same_training(a, b, ["recon_loss", "kl_loss"])
    assert a.best_val_loss == b.best_val_loss


def test_default_off_builds_no_pool_and_an_ineligible_loader_keeps_the_host_path(monkeypatch):
    images = _k255(32, 4)
    seq = DataLoader(TensorDataset(images, torch.zeros(32)), batch_size=16, shuffle=False)     # not eligible: no shuffling
    on = _gan("ns", seq)
    on.device_dataset = True
    on.train(num_epochs=2)
    assert on._pool is None
    monkeypatch.setattr(DevicePool, "from_loader", staticmethod(lambda *a, **k: pytest.fail("the default builds no pool")))
    off = _gan("ns", seq)
    off.train(num_epochs=2)
    assert getattr(off, "_pool", None) is None
    _same_training(on, off, ["Dlosses", "Glosses"])
    val = DataLoader(TensorDataset(_k255(16, 2), torch.zeros(16)), batch_size=16, shuffle=False)
    vae = _vae(DataLoader(TensorDataset(images, torch.zeros(32)), batch_size=16, shuffle=True), val)
    vae.train(num_epochs=1)
    assert getattr(vae, "_pool", None) is None
