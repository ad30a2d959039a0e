"""CPU tests of the per-sample noise mode: key derivation, configuration checks and the list-of-generators drop-in.
No compute call of the CUDA library is made here."""
import numpy as np
import pytest
import torch

from brepgen_b200.sampler import Cascade, CascadeConfig, per_sample_seeds, shard_batch, shard_config
from brepgen_b200.schedulers import DDPMScheduler, mix_seed, randn_generators, sample_keys, sample_seed


def test_sample_keys_are_pinned():
    """the keys are part of what a seeded run reproduces: changing the derivation changes every generated B-rep"""
    assert sample_seed(0, 0) == 0x46B73E79F0C37C00
    assert sample_seed(0, 1) == 0x5D60B960E0946BA0
    assert sample_seed(7, 1234) == 0x92DF2D8AC6921243
    k = sample_keys([sample_seed(0, 0), sample_seed(7, 1234)], 3)
    assert k.dtype == np.uint64 and [int(v) for v in k] == [0xC6D2B23544D67CC5, 0x1D92B962C0456E1C]
    assert int(sample_keys([5], 2)[0]) == mix_seed(5, 2)


def test_sample_keys_are_distinct_across_seeds_indices_and_stages():
    seeds = [sample_seed(s, i) for s in (0, 1, 2, 1000) for i in range(64)]
    assert len(set(seeds)) == len(seeds)           # neighbouring run seeds share no sample (not seed + index)
    keys = np.concatenate([sample_keys(seeds, st) for st in range(4)])
    assert len(set(int(k) for k in keys)) == keys.size
    # and none coincides with a batch-mode (seed, rank, stage) key
    batch = {mix_seed(s, r, st) for s in (0, 1, 2, 1000) for r in range(8) for st in range(4)}
    assert not batch & set(int(k) for k in keys)


def test_scheduler_keys_follow_first_index_and_explicit_seeds():
    s = DDPMScheduler()
    assert not s.per_sample_noise
    s.set_sample_keys(seed=4, first=10, stage=1)
    assert s.per_sample_noise
    k = s.sample_key_tensor(3, "cpu")
    assert k.dtype == torch.int64
    want = sample_keys([sample_seed(4, 10 + i) for i in range(3)], 1)
    assert np.array_equal(k.numpy().view(np.uint64), want)
    s.set_sample_keys(stage=1, sample_seeds=[sample_seed(4, 11), 99])
    assert np.array_equal(s.sample_key_tensor(2, "cpu").numpy().view(np.uint64), sample_keys([sample_seed(4, 11), 99], 1))
    with pytest.raises(ValueError):
        s.sample_key_tensor(3, "cpu")
    s.set_noise_seed(4, 0, 1)                       # back to the batch-wide stream
    assert not s.per_sample_noise


def test_per_sample_config_checks():
    assert per_sample_seeds(CascadeConfig(batch_size=3)) is None
    cfg = CascadeConfig(batch_size=3, seed=5, noise="per_sample", sample_base=7)
    assert per_sample_seeds(cfg) == [sample_seed(5, 7 + b) for b in range(3)]
    cfg = CascadeConfig(batch_size=2, noise="per_sample", sample_seeds=[11, 12])
    assert per_sample_seeds(cfg) == [11, 12]
    casc = Cascade({}, device="cpu")
    with pytest.raises(ValueError, match="sample_seeds"):
        casc.run(CascadeConfig(batch_size=3, noise="per_sample", sample_seeds=[1, 2]))
    with pytest.raises(ValueError, match="noise"):
        casc.run(CascadeConfig(batch_size=3, noise="per-sample"))


def test_shard_config_covers_the_global_batch():
    base = CascadeConfig(batch_size=7, seed=2, noise="per_sample", sample_base=100)
    one = per_sample_seeds(base)
    for ws in (1, 2, 3, 7):
        parts = []
        for r in range(ws):
            c = shard_config(base, 7, r, ws)
            lo, hi = shard_batch(7, r, ws)
            assert c.batch_size == hi - lo and c.sample_base == 100 + lo and c.noise == "per_sample"
            parts += per_sample_seeds(c)
        assert parts == one
    seeded = CascadeConfig(batch_size=5, noise="per_sample", sample_seeds=[9, 8, 7, 6, 5])
    assert [s for r in range(2) for s in per_sample_seeds(shard_config(seeded, 5, r, 2))] == [9, 8, 7, 6, 5]
    with pytest.raises(ValueError):
        shard_config(seeded, 6, 0, 2)


def _randn_tensor_list_branch(shape, generator, device, dtype):
    """restatement of the list branch of the reference's randn_tensor (utils.py:62-97, from diffusers)"""
    rand_device = device
    batch_size = shape[0]
    gen_device_type = generator[0].device.type
    if gen_device_type != device.type and gen_device_type == "cpu":
        rand_device = "cpu"
    shape = (1,) + shape[1:]
    latents = [torch.randn(shape, generator=generator[i], device=rand_device, dtype=dtype) for i in range(batch_size)]
    return torch.cat(latents, dim=0).to(device)


@pytest.mark.parametrize("shape", [(1, 5), (4, 7, 6), (3, 2, 5, 18)])
def test_generator_list_equals_randn_tensor(shape):
    def gens():
        return [torch.Generator().manual_seed(100 + i) for i in range(shape[0])]
    ref = _randn_tensor_list_branch(shape, gens(), torch.device("cpu"), torch.float32)
    got = randn_generators(shape, gens(), "cpu")
    assert got.dtype == torch.float32 and torch.equal(got, ref)
    # sample i depends on generator i alone
    alone = randn_generators((1,) + shape[1:], [torch.Generator().manual_seed(100 + shape[0] - 1)], "cpu")
    assert torch.equal(alone[0], got[-1])
    with pytest.raises(ValueError):
        randn_generators(shape, gens()[:-1] if shape[0] > 1 else gens() * 2, "cpu")
