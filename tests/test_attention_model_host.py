"""No GPU: the checks of tests/test_gpu_attention_fp64.py have teeth. The attention kernel's arithmetic is simulated in fp64
torch at small shapes (fp32 values held in fp64 and rounded to fp32 where the kernel rounds), and each simulated output goes
through the same checks as the kernel's: the documented arithmetic passes, and each of four plausible mistakes is rejected by
the check that is there to catch it."""
import math

import pytest
import torch

from test_gpu_attention_fp64 import (DT, LOG2E, Model, assert_stats, emulated, fp32, make_operands, probe_check,
                                     probe_operands)

C3 = 0.077119089663028717041015625       # ex2_emulated's cubic coefficient (attention.cu)


def rn32(t):
    return t.float().double()


def ex2_emulated(x, c3=C3):
    """attention.cu's ex2_emulated on fp32 values: clamp at -126, x = n + f, degree-3 polynomial for 2^f with fma steps (exact
    in fp64 here, then rounded to fp32), exponent n added."""
    x = x.clamp(min=-126.0)
    n = torch.floor(x)
    f = x - n
    p = rn32(fp32(c3) * f + fp32(0.227564394474029541015625))
    p = rn32(p * f + fp32(0.695146143436431884765625))
    p = rn32(p * f + 1.0)
    return torch.ldexp(p, n)


def simulate(q, k, v, B, H, Lq, Lk, D, scale, bkv, dt, emu_t=0, round_p=None, drop_last=False, c3=C3):
    """The serial schedule of attention_wgmma_kernel: fp32 logits, per key block the running maximum, P = 2^x in fp32 (MUFU
    taken as correctly rounded, or the polynomial on the pairs `emulated` selects), P rounded to E (round_p overrides),
    l += unrounded P, O += P V in fp32, O and l rescaled by alpha, out = E(O * (1 / l))."""
    E = DT[dt]
    round_p = round_p or (lambda e: e.to(E).double())
    sl2 = float(torch.tensor(fp32(scale), dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))
    nblk = -(-Lk // bkv)
    rows = torch.arange(Lq).view(-1, 1)
    out = torch.empty(B * Lq, H * D, dtype=E)
    for b in range(B):
        for h in range(H):
            cs = slice(h * D, (h + 1) * D)
            qb, kb, vb = (t[b * L:(b + 1) * L, cs].double() for t, L in ((q, Lq), (k, Lk), (v, Lk)))
            s = rn32(qb @ kb.t())
            m = torch.full((Lq, 1), -math.inf, dtype=torch.float64)
            l = torch.zeros(Lq, 1, dtype=torch.float64)
            o = torch.zeros(Lq, D, dtype=torch.float64)
            for j in range(nblk):
                keys = torch.arange(j * bkv, min(Lk, (j + 1) * bkv))
                if drop_last and j == nblk - 1:
                    keys = keys[:-1]
                sj = s[:, keys]
                m_new = torch.maximum(m, rn32(sj.amax(1, keepdim=True) * sl2))
                alpha = rn32(torch.exp2(m - m_new))
                m = m_new
                l, o = rn32(l * alpha), rn32(o * alpha)
                x = rn32(sj * sl2 - m)
                e = torch.where(emulated(emu_t, bkv, rows, keys.view(1, -1)), ex2_emulated(x, c3), rn32(torch.exp2(x)))
                l = rn32(l + e.sum(1, keepdim=True))
                o = rn32(o + round_p(e) @ vb[keys])
            out[b * Lq:(b + 1) * Lq, cs] = (o * rn32(1 / l)).to(E)
    return out


def _truncate_bf16(e):
    return (e.float().view(torch.int32) & ~0xFFFF).view(torch.float32).double()


def _cases(dt):
    """(B, H, Lq, Lk, scale, pattern, bkv): ragged key blocks, a rising and a descending maximum, both scales."""
    return [(3, 2, 96, 77, 0.125, "random", 128), (3, 2, 80, 300, 512 ** -0.5, "rising", 128),
            (2, 2, 64, 200, 0.125, "descending", 128), (3, 1, 90, 90, 512 ** -0.5, "random", 64)]


def _run(dt, **mutation):
    """Simulate every case, apply the hard bound to each, and return the pooled statistics."""
    acc = torch.zeros(4, dtype=torch.float64)
    for i, (B, H, Lq, Lk, scale, pat, bkv) in enumerate(_cases(dt)):
        D = 64
        q, k, v = make_operands(dt, B, H, Lq, Lk, D, scale, pat, 50 + i, bkv, device="cpu")
        model = Model(q, k, v, B, H, Lq, Lk, D, scale, bkv, dt)
        got = simulate(q, k, v, B, H, Lq, Lk, D, scale, bkv, dt, **mutation)
        model.check_hard(got, mutation.get("emu_t", 0) > 0, f"simulated {dt} {pat} Lk={Lk}")
        acc += model.stats(got)
    return acc


@pytest.mark.parametrize("emu_t", [0, 2])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_documented_arithmetic_is_accepted(dt, emu_t):
    """P rounded to E with round-to-nearest-even relative to the running block maximum, fp32 l, output rounded once: inside the
    hard bound, rms(z) and beta of both kernels' constants."""
    acc = _run(dt, emu_t=emu_t)
    assert_stats(acc, ("h64", dt), f"documented arithmetic {dt} emu={emu_t}")
    if dt == "bf16":
        assert_stats(acc, ("1h", dt), f"documented arithmetic {dt} emu={emu_t}")


def test_truncated_p_is_rejected_by_beta():
    """Truncating P to bf16 loses half an ulp on average (~2.8e-3 relative) in the numerator only: every output shrinks."""
    acc = torch.zeros(4, dtype=torch.float64)
    for i, (B, H, Lq, Lk, scale, pat, bkv) in enumerate(_cases("bf16")):
        q, k, v = make_operands("bf16", B, H, Lq, Lk, 64, scale, pat, 50 + i, bkv, device="cpu")
        acc += Model(q, k, v, B, H, Lq, Lk, 64, scale, bkv, "bf16").stats(
            simulate(q, k, v, B, H, Lq, Lk, 64, scale, bkv, "bf16", round_p=_truncate_bf16))
    with pytest.raises(AssertionError, match="beta"):
        assert_stats(acc, ("h64", "bf16"), "truncated P")


def test_fp16_p_rounded_at_bf16_precision_is_rejected_by_rms_z():
    acc = torch.zeros(4, dtype=torch.float64)
    for i, (B, H, Lq, Lk, scale, pat, bkv) in enumerate(_cases("fp16")):
        q, k, v = make_operands("fp16", B, H, Lq, Lk, 64, scale, pat, 50 + i, bkv, device="cpu")
        acc += Model(q, k, v, B, H, Lq, Lk, 64, scale, bkv, "fp16").stats(
            simulate(q, k, v, B, H, Lq, Lk, 64, scale, bkv, "fp16", round_p=lambda e: e.to(torch.bfloat16).double()))
    with pytest.raises(AssertionError, match=r"rms\(z\)"):
        assert_stats(acc, ("h64", "fp16"), "fp16 P at bf16 precision")


@pytest.mark.parametrize("Lk,bkv", [(77, 128), (200, 128), (90, 64)])
def test_dropped_last_key_of_a_ragged_block_is_rejected_by_the_hard_bound(Lk, bkv):
    """A mask off by one at kv_valid (`>=` where `>` belongs) loses the last valid key of the ragged block."""
    B, H, Lq = 3, 2, 64
    q, k, v = make_operands("bf16", B, H, Lq, Lk, 64, 0.125, "random", 60, bkv, device="cpu")
    model = Model(q, k, v, B, H, Lq, Lk, 64, 0.125, bkv, "bf16")
    model.check_hard(simulate(q, k, v, B, H, Lq, Lk, 64, 0.125, bkv, "bf16"), False, "documented")
    with pytest.raises(AssertionError, match="out of bound"):
        model.check_hard(simulate(q, k, v, B, H, Lq, Lk, 64, 0.125, bkv, "bf16", drop_last=True), False, "dropped key")


def _probe(dt, emu_t, max_first, c3=C3, n=4096, bkv=128, D=64, scale=0.125):
    q, k, v, ib, x = probe_operands(dt, D, scale, n, bkv, max_first, 180 + max_first, device="cpu")
    Lk = 2 * bkv
    got = simulate(q, k[:Lk], v[:Lk], 1, 1, n, Lk, D, scale, bkv, dt, emu_t=emu_t, c3=c3)[:, 0]
    rows = torch.arange(n)
    emu_rows = emulated(emu_t, bkv, rows, torch.full_like(rows, ib))
    return probe_check(got, x, dt, max_first, emu_rows, f"simulated probe {dt} emu={emu_t} max first={max_first} c3={c3}")


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_two_key_probe_accepts_the_documented_arithmetic(dt):
    for emu_t in (0, 2, 4):
        for max_first in (True, False):
            _probe(dt, emu_t, max_first)


def test_cubic_coefficient_off_by_1e_3_is_rejected_by_the_probe_mean_error():
    with pytest.raises(AssertionError, match="mean relative error"):
        _probe("bf16", 4, True, c3=C3 + 1e-3)
    with pytest.raises(AssertionError, match="mean relative error"):
        _probe("bf16", 2, True, c3=C3 + 1e-3)
    with pytest.raises(AssertionError, match="mean relative error"):
        _probe("fp16", 2, True, c3=C3 + 1e-3)
