"""The conv path's device-resident 8-bit training set (gm_b200.dcgan.DevicePool) without a GPU: packing is lossless against
the bf16 values stage_images makes (NHWC order, signed zeros kept apart), the loaders that are not eligible give None, a pool
is reused only for the same tensor and batching, and the on-device permutation's host twin gives the batch schedules the
trainers draw: distinct rows inside a GAN batch, every row once per VAE epoch."""
import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader, RandomSampler, TensorDataset, WeightedRandomSampler

from gm_b200.dcgan import DevicePool

BIG = 1 << 40                                   # a budget no test dataset reaches


def _values(kind, shape, g):
    k = torch.randint(0, 256, shape, generator=g)
    if kind == "binary":
        return (k < 77).float()
    if kind == "k255":
        return k.float() / 255
    if kind == "normalised":
        return (k.float() / 255 - 0.5) / 0.5
    # signed zeros next to a few other values: -0.0 and +0.0 must stay distinct codes
    return torch.tensor([0.0, -0.0, 1.0, -1.0, 0.5])[k % 5]


def _nhwc_bf16_bits(images, ch):
    n = images.shape[0]
    return images.float().view(n, ch, 64, 64).permute(0, 2, 3, 1).to(torch.bfloat16).contiguous().view(torch.int16).reshape(n, -1)


@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("kind", ["binary", "k255", "normalised", "signed_zero"])
def test_pack_is_bit_exact_in_nhwc_order(kind, ch):
    g = torch.Generator().manual_seed(ch)
    images = _values(kind, (7, ch * 4096), g)
    codes, table = DevicePool.pack(images, ch, chunk_rows=3)         # three chunks, the last one partial
    assert codes.dtype == torch.uint8 and codes.shape == (7, 4096 * ch) and table.shape == (256,)
    assert torch.equal(table[codes.long()], _nhwc_bf16_bits(images, ch))
    if kind == "signed_zero":
        assert len(set(table[codes.long()].unique().tolist())) == 5     # 0x0000 and 0x8000 both present
    # the [n, ch, 64, 64] layout packs to the same codes
    c2, t2 = DevicePool.pack(images.view(7, ch, 64, 64), ch)
    assert torch.equal(t2[c2.long()], _nhwc_bf16_bits(images, ch))


def _loader(images, **kw):
    kw.setdefault("batch_size", 4)
    return DataLoader(TensorDataset(images, torch.zeros(images.shape[0])), **kw)


def test_ineligible_loaders_give_none():
    g = torch.Generator().manual_seed(0)
    images = _values("k255", (6, 4096), g)
    assert DevicePool.from_loader(_loader(images, shuffle=True), 1, budget=BIG) is not None
    # 257 distinct bf16 values (the integers 0..256 are exact in bf16)
    many = torch.arange(6 * 4096).remainder(257).float().view(6, 4096)
    assert DevicePool.pack(many, 1) is None
    assert DevicePool.from_loader(_loader(many, shuffle=True), 1, budget=BIG) is None
    assert DevicePool.pack(many[:, :] % 256, 1) is not None
    # not a TensorDataset, not a DataLoader, no shuffling, other samplers, a different image size, over the budget
    assert DevicePool.from_loader(DataLoader([(x, 0) for x in images], batch_size=4, shuffle=True), 1, budget=BIG) is None
    assert DevicePool.from_loader([(images[:4], torch.zeros(4))], 1, budget=BIG) is None
    assert DevicePool.from_loader(_loader(images, shuffle=False), 1, budget=BIG) is None
    w = WeightedRandomSampler(torch.ones(6), 6)
    assert DevicePool.from_loader(_loader(images, sampler=w), 1, budget=BIG) is None
    assert DevicePool.from_loader(_loader(images, sampler=RandomSampler(images, replacement=True)), 1, budget=BIG) is None
    assert DevicePool.from_loader(_loader(images, sampler=RandomSampler(images, num_samples=4)), 1, budget=BIG) is None
    assert DevicePool.from_loader(_loader(images, shuffle=True), 3, budget=BIG) is None
    assert DevicePool.from_loader(_loader(images, shuffle=True), 1, budget=6 * 4096 - 1) is None
    assert DevicePool.from_loader(_loader(images, shuffle=True), 1, budget=6 * 4096) is not None


def test_a_pool_is_reused_for_the_same_tensor_and_batching():
    g = torch.Generator().manual_seed(1)
    images = _values("binary", (10, 4096), g)
    pool = DevicePool.from_loader(_loader(images, shuffle=True), 1, budget=BIG)
    assert (pool.n, pool.row_vals, pool.batch_size, pool.drop_last, len(pool)) == (10, 4096, 4, False, 3)
    assert DevicePool.from_loader(_loader(images, shuffle=True), 1, pool, budget=BIG) is pool        # a new loader, same tensor
    for kw in (dict(batch_size=5), dict(drop_last=True)):
        other = DevicePool.from_loader(_loader(images, shuffle=True, **kw), 1, pool, budget=BIG)
        assert other is not pool and other is not None
    assert len(DevicePool.from_loader(_loader(images, shuffle=True, drop_last=True), 1, budget=BIG)) == 2
    copy = DevicePool.from_loader(_loader(images.clone(), shuffle=True), 1, pool, budget=BIG)       # equal values, another tensor
    assert copy is not pool and torch.equal(copy.codes, pool.codes)
    assert DevicePool.from_loader(_loader(images, shuffle=False), 1, pool, budget=BIG) is None


def _pool(n, batch_size, drop_last=False):
    return DevicePool(torch.zeros(n, 16, dtype=torch.uint8), torch.zeros(256, dtype=torch.int16), 1, batch_size, drop_last, None)


def test_gan_draws_are_distinct_rows_and_change_every_step():
    pool = _pool(1000, 64)
    seed = 1234 * 1000003 ^ DevicePool.SEED_MIX
    draws = [pool.indices_host(seed, step, 0, 64).tolist() for step in range(8)]
    for d in draws:
        assert len(set(d)) == 64 and min(d) >= 0 and max(d) < 1000
    assert len({tuple(d) for d in draws}) == 8
    full = pool.indices_host(seed, 3, 0, 1000)
    assert sorted(full.tolist()) == list(range(1000))                  # a permutation; batch 0 is its prefix
    assert full[:64].tolist() == draws[3]
    assert pool.indices_host(seed + 1, 3, 0, 64).tolist() != draws[3]  # another rank's seed draws another batch


class _StubEngine:
    """stage_pool returns the drawn pool rows (their host twin) instead of staging them"""

    def stage_pool(self, pool, n, seed, round, offset=0, idx_out=None):
        return pool.indices_host(seed, round, offset, n)


@pytest.mark.parametrize("drop_last", [False, True])
def test_vae_epoch_schedule_covers_every_row_once(drop_last):
    import dc_vae as M
    N, B = 1000, 64
    loader = DataLoader(TensorDataset(torch.zeros(N, 1), torch.zeros(N)), batch_size=B, shuffle=True, drop_last=drop_last)
    model = M.DCVAE(image_size=64 * 64 * 3, hidden_dim=16, z_dim=20)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCVAETrainer(model, loader, it, it)
    assert tr.device_dataset is False
    pool = _pool(N, B, drop_last)
    epochs = []
    for e in range(2):
        tr.num_epochs = e
        batches = [(idx, n) for idx, n in tr._pool_batches(_StubEngine(), pool, 99)]
        assert len(batches) == len(loader) == (15 if drop_last else 16)
        assert all(n == B for _, n in batches[:15]) and all(len(idx) == n for idx, n in batches)
        rows = torch.cat([idx for idx, _ in batches]).tolist()
        if drop_last:
            assert len(set(rows)) == 15 * B
        else:
            assert batches[-1][1] == N - 15 * B and sorted(rows) == list(range(N))
        epochs.append(rows)
    assert epochs[0] != epochs[1]                                       # a fresh permutation per epoch
    assert np.array_equal(np.array(epochs[0][:B]), _StubEngine().stage_pool(pool, B, 99 ^ DevicePool.SEED_MIX, 0).numpy())


def test_trainers_default_to_the_host_loader():
    import dc_gan
    import dc_vae
    assert dc_gan.DCGANTrainer.device_dataset is False and dc_vae.DCVAETrainer.device_dataset is False
