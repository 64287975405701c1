"""Models of the FP8 attention (supir_attention_quant_fp8 + supir_attention_fp8, the fp8_attention option): the operand pass
in torch (its codes and scales are torch's e4m3 cast of the same fp32 values), the fp64 reference and error model of the
kernel, and a simulation of the kernel's documented arithmetic for tests/test_fp8_attention_host.py.

The kernel's arithmetic (attention_fp8.cu): logits in log2 units t = acc * sl2 with acc = q8 . k8 (exact products, fp32
accumulation) and sl2 = sq[row] * sk * fp32(scale * log2e); per 128-key block the running maximum m, p = 2^(t - m) in fp32
(MUFU or the FMA-pipe polynomial, so p <= 1), l = alpha l + sum of the unrounded p, P code = RNE_satfinite_e4m3(2^8 p),
O = alpha O + P code * v8 (vt8 in the permuted key order; the block's product on the tensor cores, the merge in fp32) with
alpha = 2^(m_old - m_new); out = bf16(O * sv[d] * (1 / (2^8 l))).

The fp64 model follows test_gpu_attention_fp64.Model with the e4m3 operands dequantized exactly and the rounding of P
replaced by a_j = ulp_e4m3(2^8 ph_j (1 + rho_j)) / 2^9: the hard bound, the noise z and the bias beta are computed the same
way, except that the two-sided noise check is on the value-offset columns (V columns 3..7 of every head carry +8, so there the
rounding of P in the numerator dominates the error): summing l from the rounded P cancels that error and drives z down, a
coarser rounding drives it up."""
import math

import torch
import torch.nn.functional as F

FP8 = torch.float8_e4m3fn
U = 2.0 ** -24
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634
C_ACC = 4
# e4m3 wgmma on Hopper adds the products of a k-step to the accumulator with ~14 bits of alignment precision (public DeepSeek-V3
# report, section 3.3.2), not fp32's 24: its error per k-step is held to C_ACC U_MMA of the magnitudes involved. Q K^T is two
# k-steps; P V four per key block, merged into O in fp32 (O = alpha O + block).
U_MMA = 2.0 ** -12
EPS_EXP = 8.8e-5                 # the polynomial's bound (MUFU's 2^-22 is smaller); covers every split of the exponentials
P_SCALE = 256.0
BKV = 128
OFFSET_COLS = slice(3, 8)        # value columns of every head that carry the +8 offset (make_operands)


def key_of_position(pos):
    """The key stored at k position `pos` of a 32-key group of vt8: 16 a + 4 c + i -> 16 a + 2 c + (i & 1) + 8 (i >> 1)."""
    a, r = pos // 16, pos % 16
    c, i = r // 4, r % 4
    return 16 * a + 2 * c + (i & 1) + 8 * (i >> 1)


def permutation(ld):
    """Key index held by each of the `ld` positions of a vt8 row."""
    p = torch.arange(ld)
    return (p // 32) * 32 + key_of_position(p % 32)


def ulp_e4m3(x):
    """Spacing of e4m3 at |x| (fp64): 2^(e - 3) for |x| in [2^e, 2^(e+1)), e >= -6; 2^-9 below (subnormals, zero)."""
    a = x.double().abs()
    _, e = torch.frexp(a)
    e = torch.where(a == 0, -6.0, torch.clamp(e.double() - 1, min=-6.0))
    return torch.exp2(e - 3)


def scales(amax):
    """(scale, inverse) of e4m3_row_scale: amax / 448 and 448 / amax as IEEE fp32 divisions, both 1 for amax = 0."""
    pos = amax > 0
    fmax = torch.full_like(amax, 448.0)
    one = torch.ones_like(amax)
    return torch.where(pos, amax / fmax, one), torch.where(pos, fmax / torch.where(pos, amax, one), one)


def quant_operands(q, k, v, B, H, Lq, Lk, ld_vt=None):
    """The operand pass in torch: q8 [B*Lq, H*64] + sq [B*Lq, H], k8 [B*Lk, H*64] + sk [B, H], vt8 [B, H, 64, ld_vt] + sv
    [B, H, 64], and v8 [B*Lk, H*64] (the V codes in natural layout, for the models)."""
    ld_vt = ld_vt or -(-Lk // 16) * 16
    qf = q.float().reshape(B * Lq, H, 64)
    sq, iq = scales(qf.abs().amax(-1))
    q8 = (qf * iq[..., None]).to(FP8).reshape(B * Lq, H * 64)
    kf = k.float().reshape(B, Lk, H, 64)
    sk, ik = scales(kf.abs().amax(dim=(1, 3)))
    k8 = (kf * ik[:, None, :, None]).to(FP8).reshape(B * Lk, H * 64)
    vf = v.float().reshape(B, Lk, H, 64)
    sv, iv = scales(vf.abs().amax(1))
    v8 = (vf * iv[:, None]).to(FP8)
    perm = permutation(ld_vt).to(q.device)
    valid = perm < Lk
    vt = torch.zeros(B, H, 64, ld_vt, dtype=torch.uint8, device=q.device)
    vt[..., valid] = v8.view(torch.uint8).permute(0, 2, 3, 1)[..., perm[valid]]
    return q8, sq.contiguous(), k8, sk.contiguous(), vt.view(FP8), sv.contiguous(), v8.reshape(B * Lk, H * 64)


def dequant(q8, sq, k8, sk, v8, sv, B, H, Lq, Lk):
    """fp64 Q, K, V [rows, H*64] of the codes and scales."""
    qd = (q8.double().view(B * Lq, H, 64) * sq.double()[..., None]).view(B * Lq, H * 64)
    kd = (k8.double().view(B, Lk, H, 64) * sk.double()[:, None, :, None]).view(B * Lk, H * 64)
    vd = (v8.double().view(B, Lk, H, 64) * sv.double()[:, None]).view(B * Lk, H * 64)
    return qd, kd, vd


def make_operands(B, H, Lq, Lk, scale, pattern, seed, device="cuda"):
    """bf16 q, k, v as column slices of one fused buffer with sentinels and poisoned next-batch keys
    (test_gpu_attention_fp64.make_operands), plus the value offset on OFFSET_COLS."""
    from test_gpu_attention_fp64 import make_operands as base
    q, k, v = base("bf16", B, H, Lq, Lk, 64, scale, pattern, seed, BKV, device=device)
    vv = v.view(B * Lk, H, 64)
    vv[:, :, OFFSET_COLS] += 8.0
    return q, k, v


class Model:
    """fp64 reference and error model of one supir_attention_fp8 launch from the exact e4m3 operands, all query rows."""

    def __init__(self, q8, sq, k8, sk, v8, sv, B, H, Lq, Lk, scale):
        qd, kd, vd = dequant(q8, sq, k8, sk, v8, sv, B, H, Lq, Lk)
        dev = qd.device
        sc = float(torch.tensor(scale, dtype=torch.float32))
        nblk = -(-Lk // BKV)
        self.B, self.Lq, self.H = B, Lq, H
        C = H * 64
        self.ref, self.fixed, self.e2, self.d2, self.var, self.d1 = (torch.empty(B * Lq, C, dtype=torch.float64, device=dev)
                                                                      for _ in range(6))
        n_o = nblk + 2                               # fp32: the merges O = alpha O + block, the products with sv and 1 / (2^8 l)
        n_l = nblk * (BKV // 8 + 2) + 6
        for b in range(B):
            for h in range(H):
                cs = slice(h * 64, (h + 1) * 64)
                qb, kb, vb = qd[b * Lq:(b + 1) * Lq, cs], kd[b * Lk:(b + 1) * Lk, cs], vd[b * Lk:(b + 1) * Lk, cs]
                rs = slice(b * Lq, (b + 1) * Lq)
                S = qb @ kb.t() * sc
                mrun = F.pad(S, (0, nblk * BKV - Lk), value=-math.inf).view(-1, nblk, BKV).amax(-1)
                mrun = mrun.cummax(1).values.repeat_interleave(BKV, 1)[:, :Lk]
                m = mrun[:, -1:]
                ph = torch.exp(S - mrun)
                gsc = torch.exp(mrun - m)
                Z = (ph * gsc).sum(1, keepdim=True)
                p = ph * gsc / Z
                V = torch.cat([vb, vb.abs(), vb * vb], 1)
                pv = p @ V
                ref = pv[:, :64]
                A = qb.norm(dim=1, keepdim=True) * kb.norm(dim=1)
                dx = sc * LOG2E * C_ACC * 2 * U_MMA * (A + A.amax(1, keepdim=True)) + 2.0 ** -21 * LOG2E * (S.abs() + mrun.abs())
                hi = ph * (1 + EPS_EXP + LN2 * dx)
                a = ulp_e4m3(P_SCALE * hi) / (2 * P_SCALE)
                pdx = p * dx
                dd = pdx @ torch.cat([vb, vb * vb], 1)
                d1 = pdx.sum(1, keepdim=True)
                self.ref[rs, cs] = ref
                self.fixed[rs, cs] = ((a * gsc / Z) @ vb.abs() + C_ACC * (4 * U_MMA + U * n_o) * pv[:, 64:128]
                                      + 1.01 * U * n_l * ref.abs())
                self.e2[rs, cs] = (pv[:, 128:] - ref * ref).clamp(min=0)
                self.d1[rs, cs] = d1.expand(-1, 64)
                self.d2[rs, cs] = (dd[:, 64:] - 2 * ref * dd[:, :64] + ref * ref * d1).clamp(min=0)
                w2 = torch.where(ph == 1, 0.0, (gsc / Z) ** 2 * (ulp_e4m3(P_SCALE * ph) / P_SCALE) ** 2 / 12)
                self.var[rs, cs] = w2 @ (vb * vb) + ulp_bf16(ref) ** 2 / 12 + (U_MMA * pv[:, 64:128]) ** 2

    def bound(self):
        return self.fixed + torch.sqrt((EPS_EXP + LN2 * self.d1) * (EPS_EXP * self.e2 + LN2 * self.d2))

    def check_hard(self, got, what):
        g = got.double()
        tol = ulp_bf16(self.ref) + self.bound()
        bad = ~((g - self.ref).abs() <= tol)
        nbad = int(bad.sum())
        if nbad:
            i = int(bad.flatten().nonzero()[0])
            raise AssertionError(f"{what}: {nbad} of {g.numel()} elements out of bound; first at {i}: got {g.flatten()[i].item()!r} "
                                 f"ref {self.ref.flatten()[i].item()!r} tol {tol.flatten()[i].item():.3g}")

    def stats(self, got):
        """[sum z^2, count, sum (got - ref) ref, sum ref^2, sum z^2 and count on the offset columns]."""
        d = got.double() - self.ref
        z = d / self.var.sqrt()
        zo = z.view(-1, self.H, 64)[:, :, OFFSET_COLS]
        return torch.tensor([float((z * z).sum()), z.numel(), float((d * self.ref).sum()), float((self.ref * self.ref).sum()),
                             float((zo * zo).sum()), zo.numel()], dtype=torch.float64)


def ulp_bf16(x):
    a = x.double().abs()
    _, e = torch.frexp(a)
    e = torch.where(a == 0, -126.0, torch.clamp(e.double() - 1, min=-126.0))
    return torch.exp2(e - 7)


# Noise and bias bounds, from one H100 run (largest measured over the kernel test's cases, in brackets) with margin. The noise
# model holds the rounding of P and of the output; the e4m3 accumulation's own noise is not in it, so over all outputs rms(z)
# only has a loose ceiling, and the two-sided check is on the offset columns, where the rounding of P dominates. The
# simulation in tests/test_fp8_attention_host.py gives 0.98 there for the documented arithmetic, 0.50 for l summed from the
# rounded P, 1.69 for P without the 2^8 scale and 13.6 for truncated P.
R_MAX = 4.0                      # all outputs (3.00)
R_OFFSET = (0.75, 1.5)           # offset columns (1.01 - 1.20)
BETA_MAX = 2.5e-3                # (-1.64e-3; truncated P: -3.8e-2, P without 2^8: -3.0e-3)


def assert_stats(acc, what):
    rms, beta, rms_o = math.sqrt(acc[0] / acc[1]), float(acc[2] / acc[3]), math.sqrt(acc[4] / acc[5])
    print(f"{what}: rms(z) = {rms:.3f}, on the offset columns {rms_o:.3f}, beta = {beta:.3e} over {int(acc[1])} outputs")
    bad = [f"rms(z) = {rms:.3f} > {R_MAX}"] if not rms <= R_MAX else []
    if not rms_o >= R_OFFSET[0]:
        bad.append(f"rms(z) on the offset columns = {rms_o:.3f} < {R_OFFSET[0]} (the rounding of P cancels against l)")
    if not rms_o <= R_OFFSET[1]:
        bad.append(f"rms(z) on the offset columns = {rms_o:.3f} > {R_OFFSET[1]} (an extra or coarser rounding of P)")
    if not abs(beta) <= BETA_MAX:
        bad.append(f"beta = {beta:.3e}, bound {BETA_MAX:.1e} (a biased rounding of P)")
    assert not bad, f"{what}: " + "; ".join(bad)
    return rms, beta, rms_o


def rn32(t):
    return t.float().double()


def simulate(q8, sq, k8, sk, vt8, sv, B, H, Lq, Lk, scale, p_scale=P_SCALE, round_p=None, l_from_rounded=False,
             perm=None):
    """The kernel's arithmetic on the CPU (MUFU taken as correctly rounded): the mutations are a different P scale, another
    rounding of 2^8 p (round_p), l summed from the rounded P, and `perm` (ld -> the key order assumed for vt8's positions)."""
    round_p = round_p or (lambda x: x.float().to(FP8).double())
    ld = vt8.shape[-1]
    perm = (perm or permutation)(ld)
    sl2_c = float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))
    nblk = -(-Lk // BKV)
    out = torch.empty(B * Lq, H * 64, dtype=torch.bfloat16)
    for b in range(B):
        for h in range(H):
            cs = slice(h * 64, (h + 1) * 64)
            qb, kb = q8[b * Lq:(b + 1) * Lq, cs].double(), k8[b * Lk:(b + 1) * Lk, cs].double()
            vcode = torch.zeros(max(Lk, int(perm.max()) + 1), 64, dtype=torch.float64)
            vcode[perm] = vt8[b, h].double().t()       # position -> the key the simulated kernel believes it holds
            sl2 = rn32(rn32(sq[b * Lq:(b + 1) * Lq, h].double() * float(sk[b, h])) * sl2_c).view(-1, 1)
            s = rn32(qb @ kb.t())
            m = torch.full((Lq, 1), -math.inf, dtype=torch.float64)
            l = torch.zeros(Lq, 1, dtype=torch.float64)
            o = torch.zeros(Lq, 64, dtype=torch.float64)
            for j in range(nblk):
                keys = torch.arange(j * BKV, min(Lk, (j + 1) * BKV))
                sj = s[:, keys]
                m_new = torch.maximum(m, rn32(sj.amax(1, keepdim=True) * sl2))
                alpha = rn32(torch.exp2(m - m_new))
                m = m_new
                l = rn32(l * alpha)
                e = rn32(torch.exp2(rn32(sj * sl2 - m)))
                pc = round_p(e * p_scale)
                l = rn32(l + (pc / p_scale if l_from_rounded else e).sum(1, keepdim=True))
                o = rn32(o * alpha + rn32(pc @ vcode[keys]))
            inv = rn32(1 / rn32(l * p_scale))
            out[b * Lq:(b + 1) * Lq, cs] = rn32(rn32(o * sv[b, h].double()) * inv).to(torch.bfloat16)
    return out
