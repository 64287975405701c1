"""No GPU: the fp8_attention option of the FP8 mode (nets.attention, ops.attention_quant_fp8 / attention_fp8). Its pack flags
and wrapper plumbing, which attentions take the FP8 path, the C ABI's argument checks, the torch model of the operand pass
(layout, key permutation, padding) and a simulation showing that the checks of tests/test_gpu_attention_fp8.py accept the
documented arithmetic and reject four plausible mistakes."""
import ctypes

import pytest
import torch

import fp8_attention_model as fm
from test_fp8_host import _record, _small_wrapper

BF = torch.bfloat16
FP8 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------------------------
# pack flags and plumbing
# ------------------------------------------------------------------------------------------------------------------
def _attn_flags(net):
    from supir_b200 import nets
    selfs = [m.attn1.fp8_attention for m in net.modules() if isinstance(m, nets.BasicTransformerBlock)]
    texts = [m.attn2.fp8_attention for m in net.modules() if isinstance(m, nets.BasicTransformerBlock)]
    zca = [m.attn.fp8_attention for m in net.modules() if isinstance(m, nets.ZeroCrossAttn)]
    return selfs, texts, zca


def test_fp8_attention_pack_flags():
    """Refused under bf16 and fp16; the plain FP8 pack leaves every attention bf16; the option marks exactly the self-attentions
    and ZeroCrossAttn, independently of fp8_convs."""
    w = _small_wrapper(FP8)
    for net in (w.diffusion_model, w.control_model):
        for dt in (BF, torch.float16):
            with pytest.raises(ValueError, match="fp8_attention"):
                net.pack(dt, fp8_attention=True)
        net.pack(FP8)
        selfs, texts, zca = _attn_flags(net)
        assert not any(selfs + texts + zca)
        for convs in (False, True):
            net.pack(FP8, fp8_convs=convs, fp8_attention=True)
            selfs, texts, zca = _attn_flags(net)
            assert selfs and all(selfs) and not any(texts) and all(zca), (selfs, texts, zca)
            assert net._fp8_convs is convs and net._fp8_attention
    assert _attn_flags(w.diffusion_model)[2], "the UNet has ZeroCrossAttn modules"
    wb = _small_wrapper(BF)
    wb.fp8_attention = True
    with pytest.raises(ValueError, match="fp8_attention"):
        wb.pack()


def test_fp8_attention_switch_invalidates_only_on_a_change():
    from supir_b200 import nets, wrappers
    w = wrappers.ControlWrapper(nets.LightGLVUNet.__new__(nets.LightGLVUNet), dtype=FP8)
    assert w.fp8_attention is False

    def arm():
        w._packed, w._plans = True, {"k": object()}

    arm()
    w.fp8_attention = 1
    assert not w._packed and not w._plans and w.fp8_attention is True
    arm()
    w.fp8_attention = True
    assert w._packed and w._plans
    w.fp8_convs = False
    assert w._packed and w._plans
    w.fp8_attention = False
    assert not w._packed and not w._plans


def test_supir_model_fp8_attention_keyword(monkeypatch):
    from supir_b200 import model as smodel

    class Wrapper(torch.nn.Module):
        def __init__(self, net):
            super().__init__()
            self.dtype = None

        def load_control_model(self, m):
            pass

    class FirstStage(torch.nn.Module):
        encoder = torch.nn.Identity()

    monkeypatch.setattr(smodel, "get_obj_from_str", lambda s: Wrapper)
    monkeypatch.setattr(smodel, "instantiate_from_config", lambda cfg: FirstStage() if cfg == "fs" else object())
    m = smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype="fp8", fp8_attention=True)
    assert m.model.dtype is FP8 and m.model.fp8_attention is True and not getattr(m.model, "fp8_convs", False)
    m = smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype="fp8")
    assert not getattr(m.model, "fp8_attention", False)
    for dt in ("bf16", "fp16", "fp32"):
        with pytest.raises(AssertionError):
            smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype=dt, fp8_attention=True)


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
class _Pool:
    def get(self, shape, dtype=BF, device=None):
        return torch.zeros(*shape, dtype=dtype)

    def put(self, *ts):
        pass


def test_self_attention_and_zerocrossattn_take_the_fp8_path(monkeypatch):
    """With the recorder in place of the C ABI: attn1.run_self and ZeroCrossAttn's run_cross issue the operand pass and the FP8
    kernel, the text cross-attention (attn2) the bf16 kernel; without the option every attention is bf16."""
    from supir_b200 import nets
    ops, calls = _record(monkeypatch)
    w = _small_wrapper(FP8)
    net = w.diffusion_model
    net.pack(FP8, fp8_attention=True)
    blk = next(m for m in net.modules() if isinstance(m, nets.BasicTransformerBlock))
    zca = next(m for m in net.modules() if isinstance(m, nets.ZeroCrossAttn))
    ctx = nets.Ctx(_Pool(), 2)
    B, L, Lk = 2, 24, 40
    a1, a2 = blk.attn1, blk.attn2
    C = a1.inner
    fp8 = ["supir_attention_quant_fp8", "supir_attention_fp8"]

    def attn_calls(fn):
        calls.clear()
        fn()
        return [c for c in calls if "attention" in c]

    xq = (torch.zeros(B * L, a1.to_q.in_features, dtype=FP8), torch.zeros(B * L))
    assert attn_calls(lambda: a1.run_self(ctx, xq, torch.zeros(B * L, C, dtype=BF), B, L)) == fp8
    k = torch.zeros(B * 77, 2 * a2.inner, dtype=BF)
    xq2 = (torch.zeros(B * L, a2.to_q.in_features, dtype=FP8), torch.zeros(B * L))
    assert attn_calls(lambda: a2.run_cross(ctx, xq2, torch.zeros(B * L, C, dtype=BF), B, L, k[:, :a2.inner], k[:, a2.inner:], 77)) == \
        ["supir_attention_bf16"]
    za = zca.attn
    kv = torch.zeros(B * Lk, 2 * za.inner, dtype=BF)
    xz = torch.zeros(B * L, za.to_q.in_features, dtype=BF)
    assert attn_calls(lambda: za.run_cross(ctx, xz, None, B, L, kv[:, :za.inner], kv[:, za.inner:], Lk, residual=False)) == fp8
    net.pack(FP8)
    assert attn_calls(lambda: a1.run_self(ctx, xq, torch.zeros(B * L, C, dtype=BF), B, L)) == ["supir_attention_bf16"]
    assert attn_calls(lambda: za.run_cross(ctx, xz, None, B, L, kv[:, :za.inner], kv[:, za.inner:], Lk, residual=False)) == \
        ["supir_attention_bf16"]


def test_ops_reject_bad_fp8_attention_calls_before_any_call(monkeypatch):
    ops, calls = _record(monkeypatch)
    B, H, Lq, Lk = 2, 2, 16, 24
    b = lambda *s: torch.zeros(*s, dtype=BF)              # noqa: E731
    q8 = lambda *s: torch.zeros(*s, dtype=FP8)            # noqa: E731
    f = lambda *s: torch.zeros(*s)                        # noqa: E731
    args = dict(q8=q8(B * Lq, 128), sq=f(B * Lq, H), k8=q8(B * Lk, 128), sk=f(B, H), vt8=q8(B, H, 64, 32), sv=f(B, H, 64))
    ops.attention_quant_fp8(b(B * Lq, 128), b(B * Lk, 128), b(B * Lk, 128), B, H, Lq, Lk, amax_ws=torch.zeros(B * H * 65, dtype=torch.int32),
                            **args)
    ops.attention_fp8(out=b(B * Lq, 128), B=B, heads=H, Lq=Lq, Lk=Lk, **args)
    assert calls == ["supir_attention_quant_fp8", "supir_attention_fp8"]
    calls.clear()
    with pytest.raises(TypeError):
        ops.attention_quant_fp8(b(B * Lq, 128).half(), b(B * Lk, 128), b(B * Lk, 128), B, H, Lq, Lk,
                                amax_ws=torch.zeros(B * H * 65, dtype=torch.int32), **args)
    with pytest.raises(TypeError):
        ops.attention_fp8(out=b(B * Lq, 128).half(), B=B, heads=H, Lq=Lq, Lk=Lk, **args)
    with pytest.raises(TypeError):
        ops.attention_fp8(out=b(B * Lq, 128), B=B, heads=H, Lq=Lq, Lk=Lk, **dict(args, k8=b(B * Lk, 128)))
    with pytest.raises(AssertionError):
        ops.attention_fp8(out=b(B * Lq, 128), B=B, heads=H, Lq=Lq, Lk=Lk, **dict(args, vt8=q8(B, H, 64, 16)))   # < Lk
    assert calls == []


# ------------------------------------------------------------------------------------------------------------------
# C ABI argument checks
# ------------------------------------------------------------------------------------------------------------------
def test_fp8_attention_entry_points_reject_bad_arguments_before_any_launch():
    from supir_b200 import _native
    lib = _native.load()
    P = lambda a: ctypes.c_void_p(a)                      # noqa: E731
    ok, ok_s = P(1 << 20), P(1 << 21)

    def quant(q=ok, ldq=640, k=ok, ldk=640, v=ok, ldv=640, q8=ok, ldq8=640, sq=ok_s, k8=ok, ldk8=640, sk=ok_s, vt8=ok, ld_vt=1024,
              sv=ok_s, amax=ok_s, B=2, H=10, Lq=1024, Lk=1024):
        rc = lib.supir_attention_quant_fp8(q, ldq, k, ldk, v, ldv, q8, ldq8, sq, k8, ldk8, sk, vt8, ld_vt, sv, amax, B, H, Lq, Lk, None)
        return rc, lib.supir_last_error()

    for kw, what in ((dict(amax=None), b"null"), (dict(vt8=None), b"null"), (dict(B=0), b"bad shape"), (dict(H=129), b"bad shape"),
                     (dict(ldq=644), b"multiples of 8"), (dict(ldv=576), b">= H * 64"), (dict(ldq8=648), b"multiples of 16"),
                     (dict(ldk8=576), b"multiples of 16"), (dict(ld_vt=1000), b"ld_vt"), (dict(ld_vt=1008), b"ld_vt"),
                     (dict(q=P((1 << 20) + 8)), b"misaligned"), (dict(vt8=P((1 << 20) + 8)), b"misaligned"),
                     (dict(sv=P((1 << 21) + 2)), b"misaligned")):
        rc, msg = quant(**kw)
        assert rc < 0 and b"supir_attention_quant_fp8" in msg and what in msg, (kw, msg)

    def attn(q8=ok, ldq=640, sq=ok_s, k8=ok, ldk=640, sk=ok_s, vt8=ok, ld_vt=1024, sv=ok_s, out=ok, ldo=640, B=2, H=10, Lq=1024,
             Lk=1024, D=64, scale=0.125):
        rc = lib.supir_attention_fp8(q8, ldq, sq, k8, ldk, sk, vt8, ld_vt, sv, out, ldo, B, H, Lq, Lk, D, scale, None)
        return rc, lib.supir_last_error()

    for kw, what in ((dict(sk=None), b"null"), (dict(out=None), b"null"), (dict(D=128), b"head_dim"), (dict(Lk=0), b"bad shape"),
                     (dict(scale=0.0), b"scale"), (dict(ldq=648), b"multiples of 16"), (dict(ldk=576), b">= H * 64"),
                     (dict(ld_vt=1020), b"ld_vt"), (dict(ld_vt=1008), b"ld_vt"), (dict(ldo=644), b"ldo"), (dict(ldo=576), b"ldo"),
                     (dict(out=P((1 << 20) + 2)), b"aligned"), (dict(sq=P((1 << 21) + 2)), b"aligned"),
                     (dict(q8=P((1 << 20) + 8)), b"16-byte aligned")):
        rc, msg = attn(**kw)
        assert rc < 0 and what in msg, (kw, msg)


# ------------------------------------------------------------------------------------------------------------------
# the operand pass model
# ------------------------------------------------------------------------------------------------------------------
def test_key_permutation_is_the_fragment_mapping():
    """Derived from the fragment layouts: the Q K^T accumulator gives thread c = lane % 4 the keys 8 t + 2 c + {0, 1} (t = 0..3
    per 32 keys), the m64k32 A fragment wants k positions 4c..4c+3 in register 0 (row r) and 16+4c..19+4c in register 2, and
    the kernel fills register 0 with t = 0, 1 and register 2 with t = 2, 3 (low half first)."""
    want = {}
    for c in range(4):
        acc_keys = [8 * t + 2 * c + e for t in range(4) for e in range(2)]     # in the order the kernel packs them
        positions = [4 * c + i for i in range(4)] + [16 + 4 * c + i for i in range(4)]
        want.update(dict(zip(positions, acc_keys)))
    got = {p: fm.key_of_position(p) for p in range(32)}
    assert got == want
    perm = fm.permutation(96)
    assert sorted(perm.tolist()) == list(range(96))           # a bijection inside every group of 32


@pytest.mark.parametrize("B,H,Lq,Lk", [(2, 3, 40, 33), (1, 2, 17, 64), (3, 1, 5, 100)])
def test_operand_pass_model_against_torch(B, H, Lq, Lk):
    """The model's codes are torch's e4m3 cast of x * (448 / amax) at the documented granularities; vt8 row (b, h, d) holds
    V[key, d]'s code at the permuted position of every key and zeros after the last key."""
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(B * L, H * 64, generator=g).to(BF) * 3 for L in (Lq, Lk, Lk))
    k[:Lk] = 0                                                                # image 0's K is all zero: scale 1
    ld = 128
    q8, sq, k8, sk, vt8, sv, v8 = fm.quant_operands(q, k, v, B, H, Lq, Lk, ld)
    for r in range(B * Lq):
        for h in range(H):
            x = q[r, h * 64:(h + 1) * 64].float()
            s = x.abs().max() / torch.tensor(448.0)
            assert float(sq[r, h]) == float(s)
            assert torch.equal(q8[r, h * 64:(h + 1) * 64].view(torch.uint8), (x * (torch.tensor(448.0) / x.abs().max())).to(FP8).view(torch.uint8))
    assert bool((sk[0] == 1).all()) and torch.equal(k8[:Lk].float(), torch.zeros(Lk, H * 64))
    for b in range(B):
        for h in range(H):
            kb = k[b * Lk:(b + 1) * Lk, h * 64:(h + 1) * 64].float()
            if b:
                assert float(sk[b, h]) == float(kb.abs().max() / torch.tensor(448.0))
            vb = v[b * Lk:(b + 1) * Lk, h * 64:(h + 1) * 64].float()
            amax = vb.abs().amax(0)
            assert torch.equal(sv[b, h], amax / torch.full_like(amax, 448.0))
            codes = (vb * (torch.full_like(amax, 448.0) / amax)).to(FP8).view(torch.uint8)     # [Lk, 64]
            row = vt8[b, h].view(torch.uint8)                                                 # [64, ld]
            for pos in range(ld):
                key = 32 * (pos // 32) + fm.key_of_position(pos % 32)
                want = codes[key] if key < Lk else torch.zeros(64, dtype=torch.uint8)
                assert torch.equal(row[:, pos], want), (b, h, pos, key)


# ------------------------------------------------------------------------------------------------------------------
# the GPU test's checks have teeth
# ------------------------------------------------------------------------------------------------------------------
CASES = [(3, 2, 96, 77, 0.125, "random"), (3, 2, 80, 300, 512 ** -0.5, "rising"), (2, 2, 64, 200, 0.125, "descending")]


def _run(**mutation):
    acc = torch.zeros(6, dtype=torch.float64)
    for i, (B, H, Lq, Lk, scale, pat) in enumerate(CASES):
        q, k, v = fm.make_operands(B, H, Lq, Lk, scale, pat, 70 + i, device="cpu")
        q8, sq, k8, sk, vt8, sv, v8 = fm.quant_operands(q, k, v, B, H, Lq, Lk)
        model = fm.Model(q8, sq, k8, sk, v8, sv, B, H, Lq, Lk, scale)
        got = fm.simulate(q8, sq, k8, sk, vt8, sv, B, H, Lq, Lk, scale, **mutation)
        model.check_hard(got, f"simulated {pat} Lk={Lk}")
        acc += model.stats(got)
    return acc


def test_documented_arithmetic_is_accepted():
    fm.assert_stats(_run(), "documented arithmetic")


def test_p_without_the_power_of_two_scale_is_rejected():
    """e4m3(p) instead of e4m3(2^8 p): probabilities below 2^-6 lose precision in the subnormals and below 2^-10 vanish."""
    with pytest.raises(AssertionError, match="coarser rounding of P"):
        fm.assert_stats(_run(p_scale=1.0), "P without 2^8")


def test_truncated_p_is_rejected():
    def trunc(x):                                         # x >= 0: round to nearest, then one code down where that went up
        c = x.float().to(FP8)
        return torch.where(c.double() > x, (c.view(torch.uint8) - 1).view(FP8).double(), c.double())

    with pytest.raises(AssertionError, match="biased rounding of P"):
        fm.assert_stats(_run(round_p=trunc), "truncated P")


def test_l_from_the_rounded_p_is_rejected():
    with pytest.raises(AssertionError, match="cancels against l"):
        fm.assert_stats(_run(l_from_rounded=True), "l from the rounded P")


def test_wrong_key_permutation_is_rejected():
    """The V codes read as if vt8 kept the natural key order: every key's probability meets another key's value."""
    with pytest.raises(AssertionError, match="out of bound"):
        _run(perm=torch.arange)
