"""CPU: the fp64 references and the acceptance rule of the attention and RMSNorm kernel tests reject subtly wrong kernels.

Each mutant below is a kernel bug that the previous tolerances let through or that nothing compared: a lost key (the newest,
the oldest, one split's partial), a read of the key the step overwrites, a read one slot past the fill, a depformer sub-step
over one key too few, an RMSNorm over dim - 1.  The mutants run on the same scenarios the GPU tests feed the kernels, and the
rules the GPU tests apply must reject every one of them, so a later loosening of a tolerance that would admit them fails here.
"""
import math

import pytest
import torch

from tests.util import (ATTN_C, Q8_FP16_C, attn_err_ratio, attn_ref64, attn_scenario, dep_scenario, rmsnorm_ref64,
                        rmsnorm_verdict, rope_ref, split_ranges)


def _ref_over(sc: dict, slots: list, k=None, v=None) -> torch.Tensor:
    """attn_ref64 over an explicit slot list per row (None = the row's valid prefix)."""
    k = sc["k_ref"] if k is None else k
    v = sc["v_ref"] if v is None else v
    out = attn_ref64(sc["q_rot"], sc["k_ref"], sc["v_ref"], sc["n_valid"])
    for b, idx in enumerate(slots):
        if idx is None:
            continue
        idx = torch.tensor(sorted(idx), dtype=torch.long)
        out[b:b + 1] = attn_ref64(sc["q_rot"][b:b + 1], k[b:b + 1, :, idx], v[b:b + 1, :, idx], [len(idx)])
    return out


def _mutants(sc: dict) -> dict:
    """kernel bug -> (its output, the rows it changes)."""
    cap, ns = sc["cap"], sc["nsplit"]
    pos, ex, nv = sc["pos"].tolist(), sc["mask"].tolist(), sc["n_valid"].tolist()
    B = sc["B"]
    full = [set(range(n)) for n in nv]
    newest = [p % cap if e else None for p, e in zip(pos, ex)]
    oldest = [(p + e) % cap if n == cap else 0 for p, e, n in zip(pos, ex, nv)]
    out = {}

    def drop(which, name):
        slots = [full[b] - {which[b]} if which[b] is not None and nv[b] > 1 else None for b in range(B)]
        out[name] = (_ref_over(sc, slots), [b for b in range(B) if slots[b] is not None])

    drop(newest, "newest key dropped")
    drop(oldest, "oldest key dropped")
    slots = []
    for b in range(B):
        rng = [r for r in split_ranges(nv[b], ns) if r[1] > r[0]]
        s0, s1 = rng[len(rng) // 2] if len(rng) > 1 else (0, 0)
        slots.append(full[b] - set(range(s0, s1)) if s1 > s0 else None)
    out["one split's partial dropped"] = (_ref_over(sc, slots), [b for b in range(B) if slots[b] is not None])
    # the executing rows attend to the key / value the step overwrites instead of the new one
    stale_k, stale_v = sc["k_ref"].clone(), sc["v_ref"].clone()
    rows = [b for b in range(B) if ex[b]]
    for b in rows:
        stale_k[b, :, pos[b] % cap] = sc["k"][b, :, pos[b] % cap]
        stale_v[b, :, pos[b] % cap] = sc["v"][b, :, pos[b] % cap]
    out["overwritten key attended"] = (attn_ref64(sc["q_rot"], stale_k, stale_v, sc["n_valid"]), rows)
    slots = [full[b] | {nv[b]} if nv[b] < cap else None for b in range(B)]
    out["one slot past n_valid"] = (_ref_over(sc, slots), [b for b in range(B) if slots[b] is not None])
    return out


SCENARIOS = [dict(H=32, cap=3000, nsplit=16), dict(H=32, cap=3000, nsplit=16, needles=False),
             dict(H=20, cap=3000, nsplit=5, needles=False), dict(H=20, cap=250, nsplit=3), dict(H=2, cap=12, nsplit=5)]


@pytest.fixture(scope="module", params=SCENARIOS, ids=lambda p: "-".join(f"{k}{v}" for k, v in p.items()))
def scenario(request):
    return attn_scenario(**request.param)


def test_reference_accepts_itself_and_rejects_every_mutant(scenario):
    sc = scenario
    want = sc["want"]
    assert torch.isfinite(want).all()
    assert attn_err_ratio(want.bfloat16(), want) <= 0.5              # the kernel's own bf16 output rounding fits twice over
    empty = sc["n_valid"] == 0
    assert empty.any() and torch.equal(want[empty], torch.zeros_like(want[empty]))
    for name, (bad, rows) in _mutants(sc).items():
        assert rows, name
        # every row the bug touches is rejected on its own, by the bf16 kernels' rule and by the 8-bit kernel's wider one
        ratios = [attn_err_ratio(bad[b].bfloat16(), want[b], c=ATTN_C + Q8_FP16_C) for b in rows]
        print(f"H={sc['H']} cap={sc['cap']} nsplit={sc['nsplit']}: {name}: smallest error / 8-bit tolerance over "
              f"{len(rows)} rows {min(ratios):.3g}")
        assert min(ratios) > 1, (name, [sc["pos"][b].item() for b, r in zip(rows, ratios) if r <= 1])


def test_old_gates_admitted_a_dropped_key():
    """Why the rule replaced the previous ones: at 3000 keys with no dominant key, losing the newest key stays inside
    rtol = atol = 2e-2 (bf16 test) and inside max < 0.1, mean < 4e-3 (8-bit test)."""
    sc = attn_scenario(H=4, cap=3000, nsplit=16, needles=False)
    bad, rows = _mutants(sc)["newest key dropped"]
    rows = [b for b in rows if sc["n_valid"][b] == 3000]
    want = sc["want"]
    err = (bad.bfloat16().double() - want).abs()[rows]
    assert torch.allclose(bad.bfloat16().double()[rows], want[rows], rtol=2e-2, atol=2e-2)
    assert err.max() < 0.1 and err.mean() < 4e-3
    assert attn_err_ratio(bad.bfloat16()[rows], want[rows]) > 1


def test_rope_reference_rounds_the_position_in_fp32():
    """Past 2^24 the fp32 position rounds to even, exactly as the kernel's (float)pos does."""
    x = torch.randn(3, 2, 128).bfloat16()
    assert torch.equal(rope_ref(x, torch.full((3,), 2 ** 24 + 3)), rope_ref(x, torch.full((3,), 2 ** 24 + 4)))
    assert not torch.equal(rope_ref(x, torch.full((3,), 2 ** 24 + 3)), rope_ref(x, torch.full((3,), 2 ** 24 + 2)))
    # at a short position the fp32 and the float64 rotation agree to bf16 rounding
    p = torch.tensor([5, 1000, 45000])
    xf = x.double().view(3, 2, 64, 2)
    freqs = torch.exp(torch.arange(64, dtype=torch.float64) * (-math.log(10000.0) * 2 / 128))
    th = freqs[None] * p.double()[:, None]
    c, s = torch.cos(th)[:, None], torch.sin(th)[:, None]
    exact = torch.stack([xf[..., 0] * c - xf[..., 1] * s, xf[..., 0] * s + xf[..., 1] * c], -1).view(3, 2, 128)
    assert ((rope_ref(x, p).double() - exact).abs() <= exact.abs() * 2 ** -7 + 1e-2).all()


@pytest.mark.parametrize("H,dep_q", [(16, 16), (2, 8)])
def test_depformer_reference_rejects_one_key_too_few(H, dep_q):
    sc = dep_scenario(3, H, dep_q)
    ks, vs = sc["k"], sc["v"]
    for s in range(1, dep_q):
        bad = attn_ref64(sc["q"][s], ks, vs, [s] * sc["B"], scale=0.125)
        r = attn_err_ratio(bad.bfloat16(), sc["want"][s])
        assert r > 1, (s, r)
    assert attn_err_ratio(sc["want"].bfloat16(), sc["want"]) <= 0.5


@pytest.mark.parametrize("dim", [4096, 2560, 1024, 256])
def test_rmsnorm_rule_rejects_the_mean_over_dim_minus_one(dim):
    g = torch.Generator().manual_seed(dim)
    x = torch.randn(130, dim, generator=g).bfloat16()
    alpha = (torch.randn(dim, generator=g) + 1).bfloat16()
    ulps, exact = rmsnorm_verdict(rmsnorm_ref64(x, alpha), x, alpha)
    assert ulps == 0 and exact == 1.0
    xd = x.double()
    bad = xd * alpha.double() / torch.sqrt(1e-8 + xd.pow(2).sum(-1, keepdim=True) / (dim - 1))
    ulps, exact = rmsnorm_verdict(bad, x, alpha)
    print(f"dim={dim}: mean over dim - 1: {exact:.4f} exact, worst {ulps:.0f} ulp")
    assert exact < 0.999
