"""Every GEMM the engine launches, checked element by element against the float64 reference of tests/gemm_reference.py:
the engine's gemm is shadowed by a checker that (1) snapshots what the call writes, runs it and bounds every output
element against float64 of the actual operands (real-data regime), and (2) replays the same call on substitute storages
of the same layout filled with integer data, where the output must equal the reference bit for bit.  Run with -s for
the census table: one row per kernel path, its calls, the worst error / bound and the integer-regime result."""
import os

import pytest
import torch

from tests import gemm_reference as G

pytestmark = pytest.mark.gpu

_SEEN = {}   # path key -> [calls, worst err / bound, integer-regime calls equal]


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


@pytest.fixture
def shadow(monkeypatch):
    _need_cuda()
    from virtex_b200 import engine as E, ops
    orig, sms = E.gemm, ops.num_sms()
    gen = torch.Generator(device="cuda").manual_seed(0)

    def checked(A, B, D, M, N, K, **kw):
        c = G.Call(A, B, D, M, N, K, **kw)
        key = G.path_key(c, sms)
        before = G.snapshot(c)
        orig(A, B, D, M, N, K, **kw)
        try:
            worst = G.check(c, before, c, sms, integer=False)
            sub = G.substitute(c)
            G.integer_fill(sub, gen)
            sb = G.snapshot(sub)
            orig(sub.A, sub.B, sub.D, M, N, K, **sub.kwargs())
            G.check(sub, sb, sub, sms, integer=True)
        except AssertionError as e:
            raise AssertionError(f"{key} M={M} N={N} K={K}: {e}") from None
        row = _SEEN.setdefault(key, [0, 0.0, 0])
        row[0] += 1
        row[1] = max(row[1], worst)
        row[2] += 1

    monkeypatch.setattr(E, "gemm", checked)
    return ops


@pytest.mark.parametrize("name", list(G.WORKLOADS))
def test_workload_gemms(shadow, name):
    G.WORKLOADS[name]("cuda")
    torch.cuda.synchronize()


def test_dynamic_schedule_and_bnr_prefetch_off(shadow, monkeypatch):
    """The dynamic tile schedule and the fused BN-backward reduction without its L2 prefetch of y."""
    monkeypatch.setenv("VTX_BNR_PREFETCH", "0")
    shadow.set_dynamic_gemm_schedule(True)
    try:
        G.WORKLOADS["r50_l1_h1024_b3"]("cuda")
        G.WORKLOADS["r50_l1_h1024_b32"]("cuda")
        torch.cuda.synchronize()
    finally:
        shadow.set_dynamic_gemm_schedule(False)


def test_batch_256_step(shadow):
    G.BATCH_256[1]("cuda")
    torch.cuda.synchronize()


def test_census_matches_the_dry_run(monkeypatch):
    """Last: the kernel paths seen above are exactly those of the dry-run census at this GPU's SM count."""
    _need_cuda()
    from tests.test_gemm_reference_cpu import census
    from virtex_b200 import ops
    sms = ops.num_sms()
    print(f"\n{'path key':<86} {'calls':>6} {'err/bound':>10} {'integer':>8}")
    for k in sorted(_SEEN):
        n, w, eq = _SEEN[k]
        print(f"{k:<86} {n:>6} {w:>10.3g} {f'{eq}/{n}':>8}")
    assert _SEEN, "no GEMM was checked"
    want = census(monkeypatch, sms)
    assert set(_SEEN) == want, (sorted(set(_SEEN) - want), sorted(want - set(_SEEN)))
