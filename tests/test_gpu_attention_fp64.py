"""The flash attention kernel (attention.cu: supir_attention_bf16 / _f16 at head_dim 64, supir_attention_1head_bf16 at 128 /
256 / 512) against an fp64 model of its rounding, on every launch path the tuning knobs reach.

The kernel's documented arithmetic (the serial schedule): S = Q K^T in fp32 on the tensor cores; per block of BKV keys the
running row maximum m, P = 2^(S * scale * log2e - m) in fp32 (MUFU.EX2 or the FMA-pipe polynomial), rounded ONCE to the
storage type E relative to that running maximum; l sums the UNROUNDED fp32 P; O += P V on the tensor cores; O and l are
rescaled by the fp32 factor alpha = ex2.approx(m_old - m_new); the output O / l is rounded to E once.

Operands are fp32 values exact in E, the reference is computed on the device in fp64. For a query row, s_j = q . k_j * scale
(exact), p_j the fp64 softmax, ph_j = exp(s_j - mrun_j) the kernel's P in its own scale (mrun_j: the fp64 running maximum up
to the block of key j, so ph_j <= 1) and ref = sum_j p_j v_j. Three checks apply to every output element:

* Hard bound (no false positives by construction):
      |got - ref| <= ulp_E(ref) + sum_j p_j |v_j| a_j / ph_j + sqrt(W1 W2)
                     + C_ACC n_o 2^-24 sum_j p_j |v_j| + 1.01 n_l 2^-24 |ref| + 2^-126 BKV max|v|
  - a_j = ulp_E(ph_j (1 + rho_j)) / 2, plus 2^-126 where ph_j < 2^-125: the rounding of P (evaluated just above ph_j, so a
    kernel value on the other side of a power of two is covered), and the flush to zero of ex2.approx.ftz / the clamp of the
    polynomial at 2^-126. l sums the unrounded P, so this error does not cancel against l: it is weighted by |v_j|, not by
    |v_j - ref|.
  - rho_j = eps_exp + ln2 dx_j: the exponential's relative error (2^-22 for MUFU, the PTX ISA's 2 ulp bound for
    ex2.approx.ftz.f32; 8.8e-5 for the polynomial) and the fp32 logit's error dx_j = scale log2e C_ACC (D / 16) 2^-24
    (A_j + max A) + 2^-22 (|t_j| + |tm_j|) in log2 units, where A_j = |q| |k_j| >= sum_d |q_d k_jd| (Cauchy-Schwarz) and t,
    tm are the logit and the running maximum in log2 units (the rounded product with the fp32 scale_log2, the fma with -m).
    These errors act on numerator and l alike, so they enter as sum_j p_j rho_j |v_j - ref|, which is bounded by Cauchy-Schwarz
    as sqrt(W1 W2) with W1 = sum_j p_j rho_j and W2 = sum_j p_j rho_j (v_j - ref)^2 (matmuls of v and v^2).
  - C_ACC = 4 bounds one wgmma k16 step: the 16 products are exact in fp32 (8- or 11-bit significands), and the tensor core's
    fp32 accumulation, which is not an IEEE-ordered sum, may truncate once when it aligns the products and once when it adds
    the accumulator: 2 x 2^-23 of the magnitudes involved. A chain of n steps is held to C_ACC n 2^-24 sum|terms|. The PV chain
    has n_o = nblk BKV / 16 steps plus nblk rescales by alpha; l is a serial fp32 sum of positive terms (n_l = nblk (BKV / 8 +
    2) + 4 roundings, the reciprocal and the final product included), a relative error on the whole output.
  - 2^-126 BKV max|v| states the assumption the masking rests on: under the polynomial a masked key (s = -inf) is clamped to
    P = 2^-126, not 0, so the keys past Lk in a ragged last block (the next batch element's rows, or TMA's zero fill) add at
    most that much. Harmless for finite values; MUFU gives exactly 0.
* Noise model: with sigma_i^2 = sum_j p_j^2 v_jc^2 ulp_E(ph_j)^2 / (12 ph_j^2) + ulp_E(ref_i)^2 / 12 (zero for the running
  maximum key itself, whose P is exactly 1) plus a small fp32-accumulation term, z_i = (got_i - ref_i) / sigma_i must have
  rms(z) <= R. Catches an extra or coarser rounding of P (P rounded twice, or the fp16 twin rounding P at bf16 precision).
* Signed multiplicative bias: beta = sum (got - ref) ref / sum ref^2, |beta| <= BETA. Truncated P shows up as ~ -2.8e-3.

All sums over keys are matmuls of the fp64 p; the bound's pieces that depend on eps_exp are kept apart so one reference serves
every path of a kernel. The CPU stand-ins of tests/cpu_ops.py meet the same hard bound on every case.
tests/test_attention_model_host.py simulates the documented arithmetic and four wrong ones on the CPU and shows that these
checks accept the first and reject each of the others.

The inputs put the kernel where it goes wrong: Lq around the 128-query CTA tile and 64-row warpgroup halves, Lk around the key
block, B = 3 so that ragged tiles of batch b read batch b+1's rows, whose keys are poisoned (tens of natural-log units above
anything in batch b, with a distinct value offset), q / k / v as column slices of one fused buffer, scales 0.125 and 512^-0.5,
outputs inside a buffer with sentinel columns on both sides and sentinel rows after B * Lq; logits random, rising by 9 log2
units in every key block (alpha << 1 each block), descending, uniform rows (q = 0) and one-hot rows whose gap to every other
key exceeds 126 log2 units."""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

import cpu_ops
from test_gpu_kernel_edges import SENTINEL, _Out, _randn, _strided, check, ulp

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634
C_ACC = 4
EPS_EXP = {False: 2.0 ** -22, True: 8.8e-5}      # some pairs emulated -> the polynomial's bound
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}

# rms(z) and |beta| bounds per (kernel, E), set from one H100 run (largest measured over every path and case of the kernel, in
# brackets) with margin. A correct kernel sits near rms(z) = 1 by construction; rounding fp16 P at bf16 precision gives ~4.8
# and truncating P gives beta ~ -2.2e-3 (the CPU simulation in tests/test_attention_model_host.py).
R = {("h64", "bf16"): 1.2,            # (0.960)
     ("h64", "fp16"): 1.2,            # (0.971)
     ("1h", "bf16"): 1.2}             # (0.999)
BETA = {("h64", "bf16"): 1e-4,        # (1.3e-6)
        ("h64", "fp16"): 1e-4,        # (1.7e-6)
        ("1h", "bf16"): 1e-4}         # (1.1e-5)
# two-key probes, per (E, rows whose exponential is MUFU / the polynomial): (|mean relative error|, fraction of the outputs
# that differ from the correctly rounded model). Measured on the H100 over all paths, in brackets; a 1e-3 error in the
# polynomial's cubic coefficient gives a mean relative error of ~2e-4 in bf16 and ~1.1e-4 in fp16.
PROBE = {("bf16", "mufu"): (5e-6, 5e-3),          # (0, 0)
         ("bf16", "emulated"): (1e-4, 5e-2),      # (6.1e-5, 2.4e-2)
         ("fp16", "mufu"): (5e-6, 5e-3),          # (6.6e-7, 7.3e-4)
         ("fp16", "emulated"): (6e-5, 1.5e-1)}    # (2.0e-5, 8.9e-2)

# A launch path: kernel ("h64" or "1h"), storage, head_dim, knob values, and the kernel template's EMU it dispatches to
Path = namedtuple("Path", "kernel dt D emu pack emu_t")
PATHS = {
    "h64-bf16": Path("h64", "bf16", 64, 0, 0, 0),
    "h64-bf16-alu2": Path("h64", "bf16", 64, 0, 2, 0),
    "h64-bf16-alu3": Path("h64", "bf16", 64, 0, 3, 0),
    "h64-bf16-alu4": Path("h64", "bf16", 64, 0, 4, 0),
    "h64-bf16-emu2": Path("h64", "bf16", 64, 2, 0, 2),
    "h64-fp16": Path("h64", "fp16", 64, 0, 0, 0),
    "h64-fp16-emu2": Path("h64", "fp16", 64, 2, 0, 2),
    "1h-128": Path("1h", "bf16", 128, 0, 0, 0),
    "1h-256": Path("1h", "bf16", 256, 0, 0, 0),
    "1h-512": Path("1h", "bf16", 512, 0, 0, 0),
    "1h-512-emu2": Path("1h", "bf16", 512, 2, 0, 2),
    "1h-512-emu4": Path("1h", "bf16", 512, 4, 0, 4),
}
SCALES = (0.125, 512 ** -0.5)


def bkv_of(kernel):
    return 128 if kernel == "h64" else 64


def emulated(emu_t, bkv, rows, key_pos):
    """Which (row, key) exponentials the kernel takes from the polynomial: pair index q = (2 t + h) & 3 with t = (key % BKV) / 8
    and h = 1 for rows 8..15 of each 16-row fragment (attention_wgmma_kernel's `emulate`)."""
    q = (2 * ((key_pos % bkv) // 8) + ((rows % 16) >= 8).long()) & 3
    if emu_t == 4:
        return torch.ones_like(q, dtype=torch.bool)
    if emu_t == 3:
        return q != 1
    if emu_t == 2:
        return (q & 1) == 1
    if emu_t == 1:
        return q == 3
    return torch.zeros_like(q, dtype=torch.bool)


def fp32(x):
    """A Python float as the kernel receives it (a C float)."""
    return float(torch.tensor(x, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def make_operands(dt, B, H, Lq, Lk, D, scale, pattern, seed, bkv, device="cuda"):
    """q [B*Lq, H*D] and k, v [B*Lk, H*D] in E, as column slices of one fused [max(B Lq, B Lk), 3 H D + 8] buffer.

    Columns 0..2 of each head are reserved: column 0 holds the poison (every query 8, batch b's keys 150 b / (8 scale), so each
    batch element's keys sit 150 natural-log units above the previous one's, a constant inside a batch element, which leaves
    its softmax unchanged; value column 0 is 4 (b + 1)); column 1 the block gain of the rising / descending patterns (even
    rows); column 2 the one-hot rows (q = 16, one hot key per batch element 100 natural-log units up, every other key <= 2)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, H, D, generator=g) * (2.5 / (math.sqrt(D) * scale))
    k = torch.randn(B, Lk, H, D, generator=g)
    v = torch.randn(B, Lk, H, D, generator=g)
    q[..., :3] = 0
    k[..., 2] = k[..., 2].clamp(max=1.0)
    if pattern in ("rising", "descending"):
        gain = 6.3 if pattern == "rising" else -3.0          # natural-log units per key block (6.3 = 9.1 log2 units)
        q[:, 0::2, :, 1] = 4.0
        k[..., 1] = ((torch.arange(Lk) // bkv).double() * gain / (4.0 * scale)).view(1, Lk, 1).float()
    else:
        assert pattern == "random", pattern
    rows = torch.arange(Lq)
    q[:, rows % 16 == 5] = 0.0                               # uniform rows
    hot = rows % 16 == 11
    q[:, hot] = 0.0
    q[:, hot, :, 2] = 16.0
    for b in range(B):
        k[b, (7 * b + 3) % Lk, :, 2] = 100.0 / (16.0 * scale)
        k[b, :, :, 0] = 150.0 * b / (8.0 * scale)
        v[b, :, :, 0] = 4.0 * (b + 1)
    q[..., 0] = 8.0
    C = H * D
    buf = torch.full((max(B * Lq, B * Lk), 3 * C + 8), SENTINEL, dtype=DT[dt])
    buf[:B * Lq, :C] = q.reshape(B * Lq, C).to(DT[dt])
    buf[:B * Lk, C:2 * C] = k.reshape(B * Lk, C).to(DT[dt])
    buf[:B * Lk, 2 * C:3 * C] = v.reshape(B * Lk, C).to(DT[dt])
    buf = buf.to(device)
    return buf[:B * Lq, :C], buf[:B * Lk, C:2 * C], buf[:B * Lk, 2 * C:3 * C]


class _OutRows(_Out):
    """_Out with SENTINEL rows after the view as well: a store past row B * Lq fails."""

    def __init__(self, rows, cols, dtype, extra_rows=3):
        super().__init__(rows + extra_rows, cols, dtype)
        self.rows = rows
        self.view[rows:] = SENTINEL
        self.view = self.full[:rows, self.lo:self.lo + cols]

    def done(self, what):
        v = super().done(what)
        assert bool((self.full[self.rows:] == SENTINEL).all()), f"{what}: wrote past the last output row"
        return v


# ------------------------------------------------------------------------------------------------------------------
# the fp64 model
# ------------------------------------------------------------------------------------------------------------------
class Model:
    """fp64 reference and error model of one launch, for query rows 0, row_step, 2 row_step, ... of each batch element.
    Tensors are [B * R, H * D]; the hard bound for a path is fixed + the exponential term of its eps_exp."""

    def __init__(self, q, k, v, B, H, Lq, Lk, D, scale, bkv, dt, row_step=1, chunk=2048):
        E = DT[dt]
        dev = q.device
        sc = fp32(scale)
        sl2 = sc * LOG2E
        nblk = -(-Lk // bkv)
        sel = torch.arange(0, Lq, row_step, device=dev)
        Rr, C = sel.numel(), H * D
        self.B, self.Lq, self.row_step, self.dt = B, Lq, row_step, dt
        self.ref, self.fixed, self.e2, self.d2, self.var = (torch.empty(B * Rr, C, dtype=torch.float64, device=dev) for _ in range(5))
        self.d1 = torch.empty(B * Rr, C, dtype=torch.float64, device=dev)
        n_o = nblk * (bkv // 16) + nblk              # PV wgmma steps (accumulator carried over blocks) + rescales
        n_l = nblk * (bkv // 8 + 2) + 4             # l: serial fp32 sum, rescales, shuffles, reciprocal, final product
        leak = 2.0 ** -126 * bkv * float(v.double().abs().max())
        for b in range(B):
            qb_all = q[b * Lq:(b + 1) * Lq][sel].double()
            kb_all, vb_all = k[b * Lk:(b + 1) * Lk].double(), v[b * Lk:(b + 1) * Lk].double()
            for h in range(H):
                cs = slice(h * D, (h + 1) * D)
                kb, vb = kb_all[:, cs], vb_all[:, cs]
                kn = kb.norm(dim=1)
                V = torch.cat([vb, vb.abs(), vb * vb], 1)
                for r0 in range(0, Rr, chunk):
                    qc = qb_all[r0:r0 + chunk, cs]
                    rs = slice(b * Rr + r0, b * Rr + r0 + qc.shape[0])
                    S = qc @ kb.t() * sc
                    mrun = F.pad(S, (0, nblk * bkv - Lk), value=-math.inf).view(-1, nblk, bkv).amax(-1)
                    mrun = mrun.cummax(1).values.repeat_interleave(bkv, 1)[:, :Lk]
                    m = mrun[:, -1:]
                    ph = torch.exp(S - mrun)                                  # the kernel's P before rounding
                    gsc = torch.exp(mrun - m)                                 # its later rescaling
                    Z = (ph * gsc).sum(1, keepdim=True)
                    p = ph * gsc / Z
                    pv = p @ V
                    ref = pv[:, :D]
                    A = qc.norm(dim=1, keepdim=True) * kn
                    dx = sl2 * C_ACC * (D // 16) * U * (A + A.amax(1, keepdim=True)) + 2.0 ** -22 * LOG2E * (S.abs() + mrun.abs())
                    hi = ph * (1 + EPS_EXP[True] + LN2 * dx)
                    a = ulp(hi, E) / 2 + torch.where(hi < 2.0 ** -125, 2.0 ** -126, 0.0)
                    pround = (a * gsc / Z) @ vb.abs()
                    pdx = p * dx
                    dd = pdx @ torch.cat([vb, vb * vb], 1)
                    d1 = pdx.sum(1, keepdim=True)
                    self.ref[rs, cs] = ref
                    self.fixed[rs, cs] = pround + C_ACC * U * n_o * pv[:, D:2 * D] + 1.01 * U * n_l * ref.abs() + leak
                    self.e2[rs, cs] = (pv[:, 2 * D:] - ref * ref).clamp(min=0)
                    self.d1[rs, cs] = d1.expand(-1, D)
                    self.d2[rs, cs] = (dd[:, D:] - 2 * ref * dd[:, :D] + ref * ref * d1).clamp(min=0)
                    w2 = torch.where(ph == 1, 0.0, (gsc / Z) ** 2 * ulp(ph, E) ** 2 / 12)
                    self.var[rs, cs] = w2 @ (vb * vb) + ulp(ref, E) ** 2 / 12 + (U * math.sqrt(n_o) * pv[:, D:2 * D]) ** 2

    def rows(self, got):
        """The modelled rows of an output [B * Lq, C]."""
        return got.reshape(self.B, self.Lq, -1)[:, ::self.row_step].reshape(-1, got.shape[-1])

    def bound(self, emulates):
        eps = EPS_EXP[emulates]
        return self.fixed + torch.sqrt((eps + LN2 * self.d1) * (eps * self.e2 + LN2 * self.d2))

    def check_hard(self, got, emulates, what):
        check(self.rows(got), self.ref, DT[self.dt], 1, self.bound(emulates), what=what)

    def stats(self, got):
        """Sums for rms(z) and beta: [sum z^2, count, sum (got - ref) ref, sum ref^2]."""
        d = self.rows(got).double() - self.ref
        z = d / self.var.sqrt()
        return torch.tensor([float((z * z).sum()), z.numel(), float((d * self.ref).sum()), float((self.ref * self.ref).sum())],
                            dtype=torch.float64)


def assert_stats(acc, key, what):
    rms, beta = math.sqrt(acc[0] / acc[1]), float(acc[2] / acc[3])
    print(f"{what}: rms(z) = {rms:.3f}, beta = {beta:.3e} over {int(acc[1])} outputs")
    bad = [f"rms(z) = {rms:.3f} > {R[key]} (an extra or coarser rounding of P)"] if not rms <= R[key] else []
    if not abs(beta) <= BETA[key]:
        bad.append(f"beta = {beta:.3e}, bound {BETA[key]:.1e} (a biased rounding of P)")
    assert not bad, f"{what}: " + "; ".join(bad)
    return rms, beta


# ------------------------------------------------------------------------------------------------------------------
# launching
# ------------------------------------------------------------------------------------------------------------------
def _lib():
    from supir_b200 import _native, ops
    return ops, _native.load()


def run(path, q, k, v, out, B, H, Lq, Lk, scale):
    """One launch of `path` with its knob values; the knobs go back to their defaults whatever happens."""
    ops, lib = _lib()
    try:
        lib.supir_set_attention_exp_emulation(path.emu)
        lib.supir_set_attention_alu_pack(path.pack)
        if path.kernel == "h64":
            ops.attention(q, k, v, out, B, H, Lq, Lk, scale)
        else:
            assert Lq == Lk and H == 1
            ops.attention_1head(q, k, v, out, B, Lq, scale)
    finally:
        lib.supir_set_attention_exp_emulation(-1)
        lib.supir_set_attention_alu_pack(-1)
    return out


def stand_in(path, q, k, v, B, H, Lq, Lk, scale):
    qc, kc, vc = (t.cpu() for t in (q, k, v))
    out = torch.empty(B * Lq, H * path.D, dtype=DT[path.dt])
    if path.kernel == "h64":
        return cpu_ops.attention(qc, kc, vc, out, B, H, Lq, Lk, scale=scale)
    return cpu_ops.attention_1head(qc, kc, vc, out, B, Lq, scale=scale)


# ------------------------------------------------------------------------------------------------------------------
# every path at the shape edges
# ------------------------------------------------------------------------------------------------------------------
def edge_cases(path):
    """(B, H, Lq, Lk, scale, key pattern): Lq around the query tile, Lk around the key block."""
    bkv = bkv_of(path.kernel)
    pats = ("random", "rising", "descending")
    if path.kernel == "h64":
        shapes = [(Lq, Lk) for Lq in (1, 63, 64, 65, 127, 128, 129) for Lk in (1, bkv - 1, bkv, bkv + 1, 77)]
        return [(3, (5, 10, 20)[i % 3], Lq, Lk, SCALES[i % 2], pats[(i // 2) % 3]) for i, (Lq, Lk) in enumerate(shapes)]
    Ls = (1, 63, 64, 65, 77, 127, 128, 129)
    return [(3, 1, L, L, s, pats[(i + j) % 3]) for i, L in enumerate(Ls) for j, s in enumerate(SCALES)]


@pytest.mark.parametrize("name", list(PATHS))
def test_attention_edges_vs_fp64_model(name):
    """Every launch path over the shape edges and logit patterns: the hard bound per element, rms(z) and beta pooled over the
    path's cases. The stand-ins meet the hard bound on the same cases."""
    path = PATHS[name]
    bkv, emulates = bkv_of(path.kernel), path.emu_t > 0
    acc = torch.zeros(4, dtype=torch.float64)
    for i, (B, H, Lq, Lk, scale, pat) in enumerate(edge_cases(path)):
        what = f"{name} B={B} H={H} Lq={Lq} Lk={Lk} scale={scale:.4g} {pat}"
        q, k, v = make_operands(path.dt, B, H, Lq, Lk, path.D, scale, pat, 1000 + i, bkv)
        model = Model(q, k, v, B, H, Lq, Lk, path.D, scale, bkv, path.dt)
        out = _OutRows(B * Lq, H * path.D, DT[path.dt])
        run(path, q, k, v, out.view, B, H, Lq, Lk, scale)
        got = out.done(what)
        model.check_hard(got, emulates, what)
        acc += model.stats(got)
        if path.emu == 0 and path.pack == 0:
            model.check_hard(stand_in(path, q, k, v, B, H, Lq, Lk, scale).to(got.device), False, "stand-in " + what)
    assert_stats(acc, (path.kernel, path.dt), name)


# ------------------------------------------------------------------------------------------------------------------
# the bench-size cases: one reference, every path of the kernel
# ------------------------------------------------------------------------------------------------------------------
BENCH = {  # kernel storage / head_dim: (B, H, Lq, Lk, query-row step of the fp64 reference)
    "h64-bf16-4096": ("bf16", 64, (2, 10, 4096, 4096, 1)),
    "h64-bf16-77": ("bf16", 64, (2, 20, 1024, 77, 1)),
    "h64-fp16-4096": ("fp16", 64, (2, 10, 4096, 4096, 1)),
    "h64-fp16-77": ("fp16", 64, (2, 20, 1024, 77, 1)),
    "1h-512-18496": ("bf16", 512, (1, 1, 18496, 18496, 4)),   # the VAE's 136^2-token tile; every 4th query row modelled
}


@pytest.mark.parametrize("case", list(BENCH))
def test_attention_bench_size_vs_fp64_model(case):
    dt, D, (B, H, Lq, Lk, step) = BENCH[case]
    paths = {n: p for n, p in PATHS.items() if p.dt == dt and p.D == D}
    kernel = next(iter(paths.values())).kernel
    bkv = bkv_of(kernel)
    scale = 0.125 if kernel == "h64" else D ** -0.5
    q, k, v = make_operands(dt, B, H, Lq, Lk, D, scale, "random", 2000, bkv)
    model = Model(q, k, v, B, H, Lq, Lk, D, scale, bkv, dt, row_step=step)
    for name, path in paths.items():
        what = f"{name} B={B} H={H} Lq={Lq} Lk={Lk}"
        out = _OutRows(B * Lq, H * D, DT[dt])
        run(path, q, k, v, out.view, B, H, Lq, Lk, scale)
        got = out.done(what)
        model.check_hard(got, path.emu_t > 0, what)
        assert_stats(model.stats(got), (kernel, dt), what)
    model.check_hard(stand_in(paths[next(iter(paths))], q, k, v, B, H, Lq, Lk, scale).to(q.device), False, f"stand-in {case}")


# ------------------------------------------------------------------------------------------------------------------
# two-key probes: the exponential and the rescale seen directly
# ------------------------------------------------------------------------------------------------------------------
def probe_operands(dt, D, scale, n, bkv, max_first, seed, device="cuda"):
    """n queries over 2 bkv keys. Key A (value 0) has logit 0, key B (value 1) logit x in (-4, 0) log2 units, spread over the
    queries; every other key is ~ -3e4 scale below. max_first: A is key 0 and B sits in block 1; otherwise B is alone in block 0
    and A sits in block 1. Returns q, k, v, B's key position, and x as the kernel computes it (fp32)."""
    E = DT[dt]
    sl2 = torch.tensor(fp32(scale), dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    q = torch.zeros(n, D)
    q[:, 1] = -torch.rand(n, generator=torch.Generator().manual_seed(seed)) * (4.0 / (8.0 * float(sl2)))
    q[:, 2] = 1.0
    q = q.to(E)
    L = 2 * bkv
    ia, ib = (0, bkv + 17) if max_first else (bkv + 17, 3)
    k = torch.zeros(max(L, n), D)
    k[:, 2] = -3e4
    k[ia, 2], k[ib, 2] = 0.0, 0.0
    k[ia, 0], k[ib, 1] = 8.0, 8.0
    v = torch.zeros(max(L, n), D)
    v[ib] = 1.0
    x = (q[:, 1].float() * 8.0) * sl2
    return q.to(device), k.to(E).to(device), v.to(E).to(device), ib, x.to(device)


def probe_model(x, dt, max_first):
    """Max key first: out = E(E(p) / (1 + p)), p = 2^x (P of key B rounded to E). Max key second: P of key B is E(1) = 1, then
    scaled by the fp32 alpha = 2^x, so out = E(alpha / (1 + alpha)) with no rounding of P."""
    E = DT[dt]
    p = torch.exp2(x.double())
    num = p.to(E).double() if max_first else p
    return (num / (1 + p)).to(E).double()


def probe_check(got, x, dt, max_first, emu_rows, what):
    """Per class of rows (key B's exponential on MUFU or on the polynomial): the mean relative error (all outputs are
    positive) and the fraction of outputs that differ from the model. With the maximum second, key B's own exponential is
    2^r of the max's rounding residual r ~ 0: exactly 1 on MUFU, but 1 - 8.5e-5 on the polynomial when r < 0 (f rounds to 1,
    the polynomial's end point), which l sums; those rows are held to the polynomial's bounds."""
    ref = probe_model(x, dt, max_first)
    rel = (got.double() - ref) / ref
    res = {}
    for cls, rows in (("mufu", ~emu_rows), ("emulated", emu_rows)):
        if bool(rows.any()):
            res[cls] = (float(rel[rows].mean()), float((got.double() != ref)[rows].double().mean()))
    print(f"{what}: " + "; ".join(f"{c}: mean rel err {m:.3g}, {f:.3g} differ from the model" for c, (m, f) in res.items()))
    for cls, (m, f) in res.items():
        bm, bf = PROBE[(dt, cls)]
        assert abs(m) <= bm, f"{what}: mean relative error {m:.3g} on the {cls} rows (bound {bm:.1e})"
        assert f <= bf, f"{what}: {f:.3g} of the {cls} rows differ from the model (bound {bf})"
    return res


@pytest.mark.parametrize("name", list(PATHS))
def test_attention_two_key_probes(name):
    """The serial schedule's documented arithmetic, seen through two keys: P rounded to E once, relative to the running
    maximum (max key first), and O and l rescaled in fp32 by the MUFU alpha with no second rounding of P (max key second)."""
    path = PATHS[name]
    bkv, D, n = bkv_of(path.kernel), path.D, 4096
    scale = 0.125 if path.kernel == "h64" else D ** -0.5
    for max_first in (True, False):
        q, k, v, ib, x = probe_operands(path.dt, D, scale, n, bkv, max_first, 180 + max_first, "cuda")
        Lk = n if path.kernel == "1h" else 2 * bkv
        k, v = k[:Lk], v[:Lk]
        out = _OutRows(n, D, DT[path.dt])
        run(path, q, k, v, out.view, 1, 1, n, Lk, scale)
        got = out.done(name)[:, 0]
        rows = torch.arange(n, device="cuda")
        emu_rows = emulated(path.emu_t, bkv, rows, torch.full_like(rows, ib))
        probe_check(got, x, path.dt, max_first, emu_rows, f"{name} max key {'first' if max_first else 'second'}")


# ------------------------------------------------------------------------------------------------------------------
# knob classes: which knob values select the same instantiation
# ------------------------------------------------------------------------------------------------------------------
def knob_class(kernel, dt, D, emu, pack):
    """The instantiation (EMU, ICVT) the dispatch picks (the table in include/supir_b200.h)."""
    if kernel == "h64":
        if emu >= 2:
            return (2, 0)
        return (0, 0) if dt == "fp16" else (0, {0: 0, 1: 2, 2: 2, 3: 3, 4: 4}[pack])
    if D == 512:
        return ({2: 2, 4: 4}.get(emu, 0), 0)
    return (0, 0)


@pytest.mark.parametrize("kd", ["h64-bf16", "h64-fp16", "1h-128", "1h-256", "1h-512"])
def test_attention_knob_classes(kd):
    """All 25 (emulation, ALU-pack) settings: outputs are bit-identical inside each class of the dispatch table, and classes
    that differ in the exponential (MUFU vs polynomial) differ somewhere in the output."""
    ops, lib = _lib()
    base = PATHS[kd]
    B, H, Lq, Lk = (3, 5, 200, 300) if base.kernel == "h64" else (2, 1, 200, 200)
    C = H * base.D
    E = DT[base.dt]
    q = _strided(_randn((B * Lq, C), 400, 1.5, E), 8)
    k = _strided(_randn((B * Lk, C), 401, 1.5, E), 16)
    v = _strided(_randn((B * Lk, C), 402, 1.0, E), 24)
    scale = 0.125 if base.kernel == "h64" else base.D ** -0.5
    outs = {}
    for emu in range(5):
        for pack in range(5):
            out = _OutRows(B * Lq, C, E)
            run(base._replace(emu=emu, pack=pack), q, k, v, out.view, B, H, Lq, Lk, scale)
            cls = knob_class(base.kernel, base.dt, base.D, emu, pack)
            got = out.done(f"{kd} emu={emu} pack={pack}").clone()
            if cls in outs:
                assert torch.equal(got, outs[cls][1]), f"{kd}: emu={emu} pack={pack} differs from {outs[cls][0]} (class {cls})"
            else:
                outs[cls] = ((emu, pack), got)
    print(f"{kd}: classes {sorted(outs)}")
    emu_classes = {}
    for cls, (_, got) in outs.items():
        emu_classes.setdefault(cls[0], got)
    keys = sorted(emu_classes)
    for i, a in enumerate(keys):
        for b in keys[i + 1:]:
            assert not torch.equal(emu_classes[a], emu_classes[b]), f"{kd}: EMU {a} and {b} give the same bits"


# ------------------------------------------------------------------------------------------------------------------
# determinism and batch invariance
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kd", ["h64-bf16", "h64-fp16", "1h-128", "1h-256", "1h-512"])
def test_attention_deterministic_and_batch_invariant(kd):
    """Two runs give the same bits, and batch elements 1..3 run alone give the bits they get inside B = 5 (DESIGN.md section 5:
    a sharded run is bit-identical to the single-GPU run)."""
    path = PATHS[kd]
    B, H, Lq, Lk = (5, 5, 129, 77) if path.kernel == "h64" else (5, 1, 129, 129)
    C, E = H * path.D, DT[path.dt]
    scale = 0.125 if path.kernel == "h64" else path.D ** -0.5
    q = _strided(_randn((B * Lq, C), 500, 1.5, E), 8)
    k = _strided(_randn((B * Lk, C), 501, 1.5, E), 8)
    v = _strided(_randn((B * Lk, C), 502, 1.0, E), 8)
    full = []
    for i in range(2):
        out = _OutRows(B * Lq, C, E)
        run(path, q, k, v, out.view, B, H, Lq, Lk, scale)
        full.append(out.done(f"{kd} run {i}"))
    assert torch.equal(full[0], full[1]), f"{kd}: two runs differ"
    part = _OutRows(3 * Lq, C, E)
    run(path, q[Lq:4 * Lq], k[Lk:4 * Lk], v[Lk:4 * Lk], part.view, 3, H, Lq, Lk, scale)
    assert torch.equal(part.done(kd), full[0][Lq:4 * Lq]), f"{kd}: batch elements 1..3 alone differ from inside B = 5"
