"""Host-side logic of the FP8 convs option of the FP8 mode (no GPU): e4m3 packing of the ResBlocks' 3x3 convolutions with one
scale per output channel, the rest of the pack equal to the FP8 linears pack, resident bytes, ControlWrapper.fp8_convs
invalidation, the SUPIRModel keyword, routing of the ops to the new entry points, and argument validation of those entry points
through the C ABI."""
import ctypes

import pytest
import torch

from test_fp8_host import _bytes, _packed_tensors, _record, _small_wrapper, _torch_quant

BF, FP8 = torch.bfloat16, torch.float8_e4m3fn


@pytest.fixture(scope="module")
def packs():
    w8 = _small_wrapper(FP8)
    w8.pack()
    wc = _small_wrapper(FP8)
    wc.fp8_convs = True
    wc.pack()
    return w8, wc


def _resblocks(net):
    from supir_b200 import nets
    return [(name, m) for name, m in net.named_modules() if isinstance(m, nets.ResBlock)]


def test_fp8_convs_pack_quantizes_the_resblock_convs(packs):
    from supir_b200 import nets
    _, wc = packs
    n = 0
    for net in (wc.diffusion_model, wc.control_model):
        assert net._fp8_linears and net._fp8_convs and net._packed_dtype == BF
        for _, m in _resblocks(net):
            assert m.fp8_convs
            for k, conv in (("_w1", m.in_layers[2]), ("_w2", m.out_layers[3])):
                q, s = getattr(m, k)
                packed = nets.pack_conv3x3(conv.weight)                      # the bf16 pack's [Cout, 9*Cin] matrix
                assert q.dtype == FP8 and q.shape == packed.shape and s.dtype == torch.float32 and s.shape == (conv.out_channels,)
                rq, rs = _torch_quant(packed)
                assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs), k
                n += 1
    assert n >= 20


def test_every_other_packed_tensor_is_the_fp8_linears_pack(packs):
    w8, wc = packs
    for n8, nc in ((w8.diffusion_model, wc.diffusion_model), (w8.control_model, wc.control_model)):
        res = {name for name, _ in _resblocks(nc)}
        t8, tc = _packed_tensors(n8), _packed_tensors(nc)
        assert set(t8) == set(tc)
        checked = 0
        for key, v in t8.items():
            if key[0] in res and key[1] in ("_w1", "_w2"):
                assert not isinstance(v, tuple) and isinstance(tc[key], tuple)
                continue
            vc = tc[key]
            for a, b in zip(v if isinstance(v, tuple) else (v,), vc if isinstance(vc, tuple) else (vc,)):
                assert (a is None and b is None) or (a.dtype == b.dtype and torch.equal(a.view(torch.uint8) if a.dtype == FP8 else a,
                                                                                          b.view(torch.uint8) if b.dtype == FP8 else b)), key
            checked += 1
        assert checked > 50


def test_packed_bytes_shrink_by_the_quantized_conv_matrices(packs):
    """bf16 [Cout, 9 Cin] (18 Cout Cin bytes) -> e4m3 (9 Cout Cin) + fp32 scales (4 Cout), for both convs of every ResBlock."""
    w8, wc = packs
    for n8, nc in ((w8.diffusion_model, wc.diffusion_model), (w8.control_model, wc.control_model)):
        want = 0
        for _, m in _resblocks(n8):
            for conv in (m.in_layers[2], m.out_layers[3]):
                want += 9 * conv.out_channels * conv.in_channels - 4 * conv.out_channels
        assert want > 0 and _bytes(n8) - _bytes(nc) == want


def test_fp8_convs_switch_invalidates_only_on_a_change():
    from supir_b200 import nets, wrappers
    w = wrappers.ControlWrapper(nets.LightGLVUNet.__new__(nets.LightGLVUNet), dtype=FP8)
    assert w.fp8_convs is False

    def arm():
        w._packed, w._plans = True, {"k": object()}

    arm()
    w.fp8_convs = True
    assert not w._packed and not w._plans and w.fp8_convs
    arm()
    w.fp8_convs = True                        # same value: nothing to drop
    assert w._packed and w._plans
    w.dtype = FP8
    assert w._packed and w._plans
    w.fp8_convs = False
    assert not w._packed and not w._plans
    arm()
    w.fp8_convs = False
    assert w._packed and w._plans


def test_fp8_convs_need_the_fp8_dtype():
    w = _small_wrapper(BF)
    w.fp8_convs = True
    with pytest.raises(ValueError, match="fp8_convs"):
        w.pack()
    net = w.diffusion_model
    for dt in (BF, torch.float16):
        with pytest.raises(ValueError, match="fp8_convs"):
            net.pack(dt, fp8_convs=True)


def test_supir_model_fp8_convs_keyword(monkeypatch):
    """fp8_convs=True with diffusion_dtype='fp8' sets the wrapper's option; any other dtype refuses it (the constructor's config
    plumbing is replaced by stubs, as in the FP8 linears test)."""
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
    m = smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype="fp8", fp8_convs=True)
    assert m.model.dtype is FP8 and m.model.fp8_convs is True
    m = smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype="fp8")
    assert m.model.dtype is FP8 and not getattr(m.model, "fp8_convs", False)
    with pytest.raises(AssertionError):
        smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype="bf16", fp8_convs=True)


def test_wrapper_fp8_convs_is_a_bool():
    from supir_b200 import nets, wrappers
    w = wrappers.ControlWrapper(nets.LightGLVUNet.__new__(nets.LightGLVUNet), dtype=FP8)
    w.fp8_convs = 1
    assert w.fp8_convs is True


def test_ops_route_fp8_conv_calls_to_the_new_entry_points(monkeypatch):
    ops, calls = _record(monkeypatch)
    q = lambda *s: torch.zeros(*s, dtype=FP8)             # noqa: E731
    f = lambda *s: torch.zeros(*s)                        # noqa: E731
    b = lambda *s: torch.zeros(*s, dtype=BF)              # noqa: E731
    i = lambda *s: torch.zeros(*s, dtype=torch.int32)     # noqa: E731
    B, H, W, Cin, Cout = 2, 4, 3, 32, 48
    ops.conv3x3_fp8(q(B * H * W, Cin), f(B), B, H, W, q(Cout, 9 * Cin), f(Cout), b(B * H * W, Cout), bias=f(Cout), rowvec=f(B, Cout))
    ops.conv3x3_fp8(q(B * H * W, Cin), f(B), B, H, W, q(Cout, 9 * Cin), f(Cout), b(B * H * W, Cout), residual=b(B * H * W, Cout))
    ops.groupnorm_apply_quant(b(B * 12, 64), B, 12, q(B * 12, 64), f(B), i(B), f(64), f(64), 1e-5, True, torch.zeros(8, dtype=torch.float64))
    assert calls == ["supir_conv3x3_fp8", "supir_conv3x3_fp8", "supir_groupnorm_apply_quant"]


def test_ops_reject_bad_fp8_conv_calls_before_any_call(monkeypatch):
    ops, calls = _record(monkeypatch)
    B, H, W, Cin, Cout = 2, 4, 3, 32, 48
    x, xs = torch.zeros(B * H * W, Cin, dtype=FP8), torch.zeros(B)
    w, ws = torch.zeros(Cout, 9 * Cin, dtype=FP8), torch.zeros(Cout)
    out = torch.zeros(B * H * W, Cout, dtype=BF)
    with pytest.raises(TypeError):
        ops.conv3x3_fp8(x.to(BF), xs, B, H, W, w, ws, out)                       # bf16 activation
    with pytest.raises(TypeError):
        ops.conv3x3_fp8(x, xs, B, H, W, w.to(BF), ws, out)                       # bf16 weight
    with pytest.raises(TypeError):
        ops.conv3x3_fp8(x, xs, B, H, W, w, ws, out.to(torch.float16))            # fp16 output
    with pytest.raises(TypeError):
        ops.conv3x3_fp8(x, xs, B, H, W, w, ws, out, residual=torch.zeros(B * H * W, Cout, dtype=torch.float16))
    with pytest.raises(TypeError):
        ops.conv3x3_fp8(x, xs.double(), B, H, W, w, ws, out)                     # fp64 scales
    with pytest.raises(ValueError):
        ops.conv3x3_fp8(x, xs, B, H, W, w, ws, out, act=2)                       # no GEGLU
    with pytest.raises(AssertionError):
        ops.conv3x3_fp8(x, torch.zeros(B * H * W), B, H, W, w, ws, out)          # per-row, not per-image, scales
    g = torch.zeros(64)
    sums = torch.zeros(8, dtype=torch.float64)
    xg, qg = torch.zeros(24, 64, dtype=BF), torch.zeros(24, 64, dtype=FP8)
    amax = torch.zeros(B, dtype=torch.int32)
    with pytest.raises(TypeError):
        ops.groupnorm_apply_quant(xg.half(), B, 12, qg, torch.zeros(B), amax, g, g, 1e-5, True, sums)
    with pytest.raises(TypeError):
        ops.groupnorm_apply_quant(xg, B, 12, qg.to(BF), torch.zeros(B), amax, g, g, 1e-5, True, sums)
    with pytest.raises(TypeError):
        ops.groupnorm_apply_quant(xg, B, 12, qg, torch.zeros(B), amax.float(), g, g, 1e-5, True, sums)
    with pytest.raises(TypeError):
        ops.groupnorm_apply_quant(xg, B, 12, qg, torch.zeros(B), amax, g, g, 1e-5, True, sums.float())
    with pytest.raises(AssertionError):
        ops.groupnorm_apply_quant(xg, B, 12, qg, torch.zeros(24), amax, g, g, 1e-5, True, sums)    # per-row scales
    assert calls == []


def test_fp8_conv_entry_points_reject_bad_arguments_before_any_launch():
    """Negative return code + message, before the device is touched (this runs without a GPU)."""
    from supir_b200 import _native
    lib = _native.load()
    P = lambda a: ctypes.c_void_p(a)                      # noqa: E731
    ok, ok_s = P(1 << 20), P(1 << 21)

    def conv(x=ok, ldx=320, xs=ok_s, Wp=ok, ws=ok_s, out=ok, ldc=320, B=2, H=8, W=8, Cin=320, Cout=320, ep=None):
        rc = lib.supir_conv3x3_fp8(x, ldx, xs, Wp, ws, out, ldc, B, H, W, Cin, Cout, ep, None)
        return rc, lib.supir_last_error()

    rc, msg = conv(x=P((1 << 20) + 8))
    assert rc < 0 and b"supir_conv3x3_fp8" in msg and b"aligned" in msg
    rc, msg = conv(Wp=P((1 << 20) + 8))
    assert rc < 0 and b"aligned" in msg
    rc, msg = conv(xs=P((1 << 21) + 2))
    assert rc < 0 and b"aligned" in msg
    rc, msg = conv(Cin=40, ldx=48)
    assert rc < 0 and b"multiples of 16" in msg
    rc, msg = conv(ldx=328)
    assert rc < 0 and b"multiples of 16" in msg
    rc, msg = conv(ldx=304)
    assert rc < 0 and b"ldx >= Cin" in msg
    rc, msg = conv(B=0)
    assert rc < 0 and b"bad shape" in msg
    rc, msg = conv(ws=None)
    assert rc < 0 and b"null" in msg
    rc, msg = conv(ldc=100)
    assert rc < 0 and b"ldc" in msg
    for field, val in (("ln_stats", 1 << 22), ("out_f32", 1), ("act", 2)):
        ep = _native.Epilogue()
        setattr(ep, field, val)
        rc, msg = conv(ep=ctypes.byref(ep))
        assert rc < 0 and b"FP8 conv epilogue" in msg, field

    def gn(x=ok, ldx=320, q=ok, ldq=320, sc=ok_s, amax=ok_s, B=2, HW=64, C=320, groups=32, sums=ok):
        rc = lib.supir_groupnorm_apply_quant(x, ldx, q, ldq, sc, amax, B, HW, C, groups, sums, ok, ok, 1e-5, 1, None)
        return rc, lib.supir_last_error()

    rc, msg = gn(C=40, ldx=40, ldq=48, groups=8)                  # C % 16
    assert rc < 0 and b"supir_groupnorm_apply_quant" in msg and b"unsupported C" in msg
    rc, msg = gn(ldq=328)                                          # ldq % 16
    assert rc < 0 and b"unsupported C" in msg
    rc, msg = gn(C=336, ldx=336, ldq=336)                          # C % groups
    assert rc < 0 and b"unsupported C" in msg
    rc, msg = gn(q=P((1 << 20) + 8))
    assert rc < 0 and b"misaligned" in msg
    rc, msg = gn(amax=P((1 << 21) + 2))
    assert rc < 0 and b"misaligned" in msg
    rc, msg = gn(sums=None)
    assert rc < 0 and b"null" in msg
    rc, msg = gn(HW=0)
    assert rc < 0 and b"bad shape" in msg
