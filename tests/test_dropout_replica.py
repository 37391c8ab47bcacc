"""CPU checks of the host dropout replica (tests/dropout_replica.py) that the head-kernel tests feed to their float64
references: the vectorised numpy form against the plain Python-integer statement, and the drop rate it implies."""
import math

import numpy as np

from tests import dropout_replica as R


def test_vectorised_replica_matches_python_integers():
    rng = np.random.default_rng(0)
    seeds = [0, 1, 5, 77, 2 ** 32 - 1, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 5, 2 ** 64 - 1, -1]
    sites = [0, 1, 5, 14, 21, 1000, 1045, 2 ** 31]
    triples = []
    for _ in range(400):
        seed = int(rng.integers(0, 2 ** 63)) * 2 + int(rng.integers(0, 2)) if rng.random() < 0.4 else \
            seeds[int(rng.integers(len(seeds)))]
        site = sites[int(rng.integers(len(sites)))]
        idx = int(rng.integers(0, 2 ** 40)) if rng.random() < 0.5 else int(rng.integers(0, 4096))
        triples.append((seed, site, idx))
    triples += [(2 ** 64 - 1, 1045, 0), (2 ** 63 + 5, 1045, 3), (1, 0, 2 ** 40 + 1)]
    for p in (0.1, 0.5, 0.0):
        for seed, site, idx in triples:
            got = float(R.keep_scale(seed, site, np.array([idx]), p)[0])
            assert got == R.keep_scale_scalar(seed, site, idx, p), (seed, site, idx, p)
    # the two's-complement int64 form of a seed is the same device word
    assert R.as_u64(R.as_i64(2 ** 63 + 5)) == 2 ** 63 + 5 and R.as_i64(2 ** 64 - 1) == -1
    # four consecutive elements share one hash, the next group uses another
    seed, site = 2 ** 63 + 5, 1045
    h0 = R.hash_u64(seed, site, np.array([0, 1], dtype=np.uint64))
    assert h0[0] != h0[1]


def test_threshold_is_computed_from_float32_p():
    assert R.threshold(0.1) == 6554            # 0.1f * 65536 = 6553.6001 -> 6554
    assert R.threshold(0.5) == 32768
    assert R.threshold(0.0) == 0
    assert R.inv_keep(0.1) == np.float32(1.0) / (np.float32(1.0) - np.float32(0.1))


def test_drop_rate_at_p_0_1():
    n = 1 << 20
    for seed, site in ((1, 0), (2 ** 63 + 5, 1045), (2 ** 64 - 1, 14)):
        s = R.flat_scale(seed, site, (n,), 0.1)
        assert set(np.unique(s).tolist()) == {0.0, float(R.inv_keep(0.1))}
        q = 6554 / 65536
        rate = float((s == 0).mean())
        assert abs(rate - q) < 4 * math.sqrt(q * (1 - q) / n), (seed, site, rate)


def test_attention_index_layout():
    idx = R.attn_index(2, 3, 5, 7)
    assert idx.shape == (2, 3, 5, 7)
    assert int(idx[1, 2, 4, 6]) == ((1 * 3 + 2) * 32 + 4) * 64 + 6
