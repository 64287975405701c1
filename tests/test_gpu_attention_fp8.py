"""The FP8 attention (fp8_attention option of the FP8 mode) on the GPU: the operand pass (supir_attention_quant_fp8) bit for bit
against torch, the kernel (supir_attention_fp8) against the fp64 model of its rounding in tests/fp8_attention_model.py, batch
independence, and the networks, the engine and graph replay with the option on and off."""
import warnings

import pytest
import torch
import torch.nn.functional as F

import fp8_attention_model as fm
from test_gpu_fp8 import FP8_LAYERS, _depth1, _engine, _fake_quant, _inputs, _oracle, _rel, _SeededNoise
from test_gpu_fp8_conv import FP8_CONVS, _fake_quant_image
from weights import randn

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FP8 = torch.float8_e4m3fn
SENT = 0x5A                      # sentinel byte around every e4m3 output
SENT_F = -7.0                    # sentinel around every fp32 scale output


def _ops():
    from supir_b200 import ops
    return ops


class _Buf:
    """A [*shape] view with sentinels around it: `pad` extra elements at the end of every row and 2 extra rows."""

    def __init__(self, rows, cols, dtype, pad=16):
        self.full = torch.empty(rows + 2, cols + pad, dtype=torch.uint8 if dtype == FP8 else dtype, device="cuda")
        self.full.fill_(SENT if dtype == FP8 else SENT_F)
        self.view = self.full[:rows, :cols]
        self.rows, self.cols, self.dtype = rows, cols, dtype
        if dtype == FP8:
            self.view = self.view.view(FP8)

    def outside_untouched(self):
        s = SENT if self.dtype == FP8 else SENT_F
        return bool((self.full[self.rows:] == s).all()) and bool((self.full[:self.rows, self.cols:] == s).all())


def run_quant(q, k, v, B, H, Lq, Lk, extra_vt=16):
    """The operand pass into sentinel-guarded buffers: q8 / k8 with 32 spare bytes per row, vt8 rows extra_vt bytes past
    attention_vt_ld(Lk), scales with spare elements. Returns the operand views and the guards."""
    ops = _ops()
    C, ld = H * 64, ops.attention_vt_ld(Lk) + extra_vt
    q8, k8 = _Buf(B * Lq, C, FP8, 32), _Buf(B * Lk, C, FP8, 32)
    vt = torch.full((B * H * 64 * ld + 64,), SENT, dtype=torch.uint8, device="cuda")
    vt8 = vt[:B * H * 64 * ld].view(FP8).view(B, H, 64, ld)
    sq, sk, sv = _Buf(B * Lq, H, torch.float32, 0), _Buf(B, H, torch.float32, 0), _Buf(B * H, 64, torch.float32, 0)
    amax = torch.empty(B * H * 65, dtype=torch.int32, device="cuda").fill_(12345)
    ops.attention_quant_fp8(q, k, v, B, H, Lq, Lk, q8.view, sq.view, k8.view, sk.view, vt8, sv.view.view(B, H, 64), amax)
    torch.cuda.synchronize()
    guards = dict(q8=q8, k8=k8, sq=sq, sk=sk, sv=sv)
    for name, g in guards.items():
        assert g.outside_untouched(), f"operand pass wrote outside {name}"
    assert bool((vt[B * H * 64 * ld:] == SENT).all()), "operand pass wrote past vt8"
    return q8.view, sq.view, k8.view, sk.view, vt8, sv.view.view(B, H, 64)


def run_attention(ops_args, B, H, Lq, Lk, scale):
    from test_gpu_attention_fp64 import _OutRows
    q8, sq, k8, sk, vt8, sv = ops_args
    out = _OutRows(B * Lq, H * 64, BF)
    _ops().attention_fp8(q8, sq, k8, sk, vt8, sv, out.view, B, H, Lq, Lk, scale)
    return out.done(f"attention_fp8 B={B} H={H} Lq={Lq} Lk={Lk}")


# ------------------------------------------------------------------------------------------------------------------
# operand pass
# ------------------------------------------------------------------------------------------------------------------
QUANT_CASES = [(3, 10, 129, 33), (2, 5, 77, 300), (1, 20, 64, 1), (2, 2, 200, 128), (3, 1, 31, 129)]


@pytest.mark.parametrize("B,H,Lq,Lk", QUANT_CASES)
def test_operand_pass_bit_identical_to_torch(B, H, Lq, Lk):
    """Codes and scales equal the torch model's (torch's e4m3 cast), vt8 is the permuted, zero-padded transpose; inputs are
    column slices of one fused buffer, Lq != Lk, nothing is written outside the outputs."""
    q, k, v = fm.make_operands(B, H, Lq, Lk, 0.125, "random", 7 + Lk)
    got = run_quant(q, k, v, B, H, Lq, Lk)
    ld = got[4].shape[3]
    want = fm.quant_operands(q, k, v, B, H, Lq, Lk, ld)
    for name, g, w in zip(("q8", "sq", "k8", "sk", "vt8", "sv"), got, want):
        if g.dtype == FP8:
            assert torch.equal(g.view(torch.uint8), w.view(torch.uint8)), name
        else:
            assert torch.equal(g, w), name


def test_operand_pass_scales_are_per_image():
    """Images 1 and 2 quantized alone give the bits they get inside a batch of 3 whose image 0 is 100x larger."""
    B, H, Lq, Lk = 3, 4, 100, 130
    q, k, v = fm.make_operands(B, H, Lq, Lk, 0.125, "random", 11)
    q, k, v = q.clone(), k.clone(), v.clone()
    for t, L in ((q, Lq), (k, Lk), (v, Lk)):
        t[:L] *= 100
    full = run_quant(q, k, v, B, H, Lq, Lk)
    part = run_quant(q[Lq:], k[Lk:], v[Lk:], 2, H, Lq, Lk)
    assert torch.equal(full[0][Lq:].view(torch.uint8), part[0].view(torch.uint8)) and torch.equal(full[1][Lq:], part[1])
    assert torch.equal(full[2][Lk:].view(torch.uint8), part[2].view(torch.uint8)) and torch.equal(full[3][1:], part[3])
    assert torch.equal(full[4][1:].view(torch.uint8), part[4].view(torch.uint8)) and torch.equal(full[5][1:], part[5])


# ------------------------------------------------------------------------------------------------------------------
# kernel against the fp64 model
# ------------------------------------------------------------------------------------------------------------------
def _kernel_case(B, H, Lq, Lk, scale, pat, seed):
    q, k, v = fm.make_operands(B, H, Lq, Lk, scale, pat, seed)
    ops_args = run_quant(q, k, v, B, H, Lq, Lk)
    q8, sq, k8, sk, vt8, sv = ops_args
    v8 = fm.quant_operands(q, k, v, B, H, Lq, Lk, vt8.shape[3])[6]
    model = fm.Model(q8, sq, k8, sk, v8, sv, B, H, Lq, Lk, scale)
    got = run_attention(ops_args, B, H, Lq, Lk, scale)
    what = f"B={B} H={H} Lq={Lq} Lk={Lk} scale={scale:.4g} {pat}"
    model.check_hard(got, what)
    return model.stats(got)


def edge_cases():
    pats = ("random", "rising", "descending")
    shapes = [(Lq, Lk) for Lq in (1, 64, 127, 128, 129) for Lk in (1, 31, 32, 33, 127, 128, 129)]
    return [(3, (10, 20)[i % 2], Lq, Lk, (0.125, 512 ** -0.5)[(i // 2) % 2], pats[i % 3]) for i, (Lq, Lk) in enumerate(shapes)]


def test_attention_fp8_edges_vs_fp64_model():
    """Lq around the query tile, Lk around the key block and the 32-key groups, B = 3 with poisoned next-batch keys, H = 10 /
    20, one-hot and uniform rows (make_operands): the hard bound per element; rms(z), its lower bound on the offset columns and
    beta pooled."""
    acc = torch.zeros(6, dtype=torch.float64)
    for i, case in enumerate(edge_cases()):
        acc += _kernel_case(*case, 3000 + i)
    fm.assert_stats(acc, "attention_fp8 edges")


@pytest.mark.parametrize("B,H,L", [(2, 10, 1024), (2, 10, 4096), (2, 20, 1024)])
def test_attention_fp8_bench_size_vs_fp64_model(B, H, L):
    fm.assert_stats(_kernel_case(B, H, L, L, 0.125, "random", 4000 + L), f"attention_fp8 B={B} H={H} L={L}")


@pytest.mark.parametrize("Lk", [64, 96])
def test_one_hot_rows_at_every_key_position(Lk):
    """Query r sees key r % 64 alone (orthogonal keys, a logit gap of 40 natural-log units): its output is that key's value row.
    Every position inside both 32-key groups is hit, so a wrong key permutation in vt8 moves outputs to another key's value."""
    B, H, Lq = 1, 2, 128
    eye = torch.eye(64)
    k = torch.zeros(Lk, 64)
    k[:64] = eye
    q = eye[torch.arange(Lq) % 64] * (40.0 / 0.125)
    v = torch.randn(Lk, 64, generator=torch.Generator().manual_seed(5)) + 2.0
    q, k, v = (t.repeat(1, H).to(BF).cuda() for t in (q, k, v))
    ops_args = run_quant(q, k, v, B, H, Lq, Lk)
    got = run_attention(ops_args, B, H, Lq, Lk, 0.125).double()
    q8, sq, k8, sk, vt8, sv = ops_args
    v8 = fm.quant_operands(q, k, v, B, H, Lq, Lk, vt8.shape[3])[6]
    vd = (v8.double().view(Lk, H, 64) * sv.double()[0][None]).view(Lk, H * 64)
    want = vd[torch.arange(Lq) % 64]
    bad = ((got - want).abs() > fm.ulp_bf16(want)).any(1)
    assert not bool(bad.any()), f"{int(bad.sum())} rows differ from their hot key's value by more than one bf16 ulp"


def test_batch_rows_independent():
    """A row computed inside a batch of 3 (operand pass + kernel) is bit-identical to the same row computed alone."""
    B, H, Lq, Lk = 3, 5, 200, 170
    q, k, v = fm.make_operands(B, H, Lq, Lk, 0.125, "random", 17)
    full = run_attention(run_quant(q, k, v, B, H, Lq, Lk), B, H, Lq, Lk, 0.125)
    one = run_attention(run_quant(q[Lq:2 * Lq], k[Lk:2 * Lk], v[Lk:2 * Lk], 1, H, Lq, Lk), 1, H, Lq, Lk, 0.125)
    assert torch.equal(full[Lq:2 * Lq], one)


# ------------------------------------------------------------------------------------------------------------------
# networks
# ------------------------------------------------------------------------------------------------------------------
def _wrapper(cfg, sd, dtype, fp8_convs, fp8_attention):
    from supir_b200 import nets, wrappers
    with torch.device("cuda"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **cfg)
        ctrl = nets.GLVControl(input_upscale=1, **cfg)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.fp8_convs, w.fp8_attention = fp8_convs, fp8_attention
    w.load_control_model(ctrl)
    w.load_state_dict(sd, strict=True)
    return w


def _fq(x, dims):
    """e4m3 fake quantization with one scale per amax over `dims`."""
    amax = x.abs().amax(dim=dims, keepdim=True)
    pos = amax > 0
    s = torch.where(pos, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
    inv = torch.where(pos, torch.full_like(amax, 448.0) / torch.where(pos, amax, torch.ones_like(amax)), torch.ones_like(amax))
    return (x * inv).to(FP8).float() * s


def _fake_sdpa(q, k, v):
    """softmax(q k^T / 8) v at the FP8 attention's quantization points, q, k, v [b, heads, n, 64] (bf16 values as stored): Q per
    (token, head), K per (image, head), V per (image, head, channel), P = e4m3(2^8 p) / 2^8 relative to the row maximum (the
    kernel's running maximum differs only in the key blocks before the one holding the maximum), l of the unrounded p."""
    q, k, v = (t.to(BF).float() for t in (q, k, v))
    qd, kd, vd = _fq(q, (3,)), _fq(k, (2, 3)), _fq(v, (2,))
    s = qd @ kd.transpose(-1, -2) * 0.125
    p = torch.exp(s - s.amax(-1, keepdim=True))
    pc = (p * 256).to(FP8).float() / 256
    return (pc @ vd) / p.sum(-1, keepdim=True)


# {fp8_convs: (fake-quantized oracle, plain oracle)}: measured on an H100 80GB HBM3 at 700 W (see DESIGN.md section 7) as
# 0.0167 / 0.0187 without and 0.0318 / 0.0379 with fp8_convs, with margin
ORACLE_BOUNDS = {False: (0.025, 0.03), True: (0.045, 0.055)}


@pytest.mark.parametrize("fp8_convs", [False, True])
def test_network_fp8_attention_vs_oracle_with_and_without_fake_quantization(monkeypatch, fp8_convs):
    from oracle import unet as ounet
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    cc = {k: v.cuda() for k, v in cond.items()}
    w = _wrapper(cfg, sd, FP8, fp8_convs, True)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        out = w(x.cuda(), t.cuda(), cc, control_scale=0.8).cpu()
    assert bool(torch.isfinite(out).all())
    plain = _oracle(sd, x, t, cond, 0.8)
    lin0, conv0, attn0 = ounet._lin, ounet._conv, ounet.attention

    def lin(sdd, p, xx):
        if ".transformer_blocks." in p and p.endswith(FP8_LAYERS):
            wq = _fake_quant(sdd[p + ".weight"].to(BF).float())
            return F.linear(_fake_quant(xx), wq, sdd.get(p + ".bias"))
        return lin0(sdd, p, xx)

    def conv(sdd, p, xx, stride=1, padding=1):
        if fp8_convs and p.endswith(FP8_CONVS):
            wt = sdd[p + ".weight"].to(BF).float()
            wq = _fake_quant(wt.reshape(wt.shape[0], -1)).reshape(wt.shape)
            return F.conv2d(_fake_quant_image(xx), wq, sdd.get(p + ".bias"), stride=stride, padding=padding)
        return conv0(sdd, p, xx, stride=stride, padding=padding)

    def attention(sdd, p, xx, context, heads):
        if not (context is None or p.endswith(".attn")):          # the text cross-attention stays bf16
            return attn0(sdd, p, xx, context, heads)
        ctx = xx if context is None else context
        q, k, v = lin(sdd, p + ".to_q", xx), lin(sdd, p + ".to_k", ctx), lin(sdd, p + ".to_v", ctx)
        b, n, c = q.shape
        sp = lambda tt: tt.view(b, -1, heads, c // heads).transpose(1, 2)      # noqa: E731
        o = _fake_sdpa(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(b, n, c)
        return lin(sdd, p + ".to_out.0", o)

    monkeypatch.setattr(ounet, "_lin", lin)
    monkeypatch.setattr(ounet, "_conv", conv)
    monkeypatch.setattr(ounet, "attention", attention)
    fake = _oracle(sd, x, t, cond, 0.8)
    ea, eb = _rel(out, fake), _rel(out, plain)
    print(f"depth-1 FP8 attention networks (fp8_convs={fp8_convs}): vs fake-quantized oracle {ea:.4g}, vs plain oracle {eb:.4g} "
          f"(|fake - plain| / |plain| = {_rel(fake, plain):.4g})")
    assert ea <= ORACLE_BOUNDS[fp8_convs][0]
    assert eb <= ORACLE_BOUNDS[fp8_convs][1]
    assert ea < eb


def test_graph_replay_and_mode_off_bit_identical():
    """fp8 -> fp8 + attention -> fp8 -> fp8 + convs + attention -> fp8 + convs: replay equals eager with the option on, and with
    it off each mode gives back its output without the option bit for bit."""
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    args = (x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()})
    w = _wrapper(cfg, sd, FP8, False, False)
    f1 = w(*args, control_scale=0.8).clone()
    w.fp8_attention = True
    assert not w._packed and not w._plans
    a1 = w(*args, control_scale=0.8).clone()
    plan = next(iter(w._plans.values()))
    assert plan.graph is not None
    plan.out.fill_(float("nan"))
    plan._run()
    torch.cuda.synchronize()
    eager = plan.out.clone()
    assert bool(torch.isfinite(eager).all()) and torch.equal(eager, a1)
    assert torch.equal(w(*args, control_scale=0.8), a1)
    assert not torch.equal(a1, f1)
    w.fp8_attention = False
    assert torch.equal(w(*args, control_scale=0.8), f1)
    w.fp8_convs = True
    c1 = w(*args, control_scale=0.8).clone()
    w.fp8_attention = True
    ca = w(*args, control_scale=0.8).clone()
    assert bool(torch.isfinite(ca).all()) and not torch.equal(ca, c1)
    w.fp8_attention = False
    assert torch.equal(w(*args, control_scale=0.8), c1)


# measured on an H100 80GB HBM3 at 700 W (see DESIGN.md section 7): 0.0234 untiled, 0.0267 tiled, with margin
ENGINE_BOUND = 0.04


@pytest.mark.parametrize("tiled", [False, True])
def test_engine_fp8_attention_end_to_end(monkeypatch, tiled):
    img = (randn((1, 3, 256, 256), 200) * 0.5).clamp(-1, 1).cuda()
    c = {"crossattn": randn((1, 77, 2048), 201).cuda(), "vector": randn((1, 2816), 202).cuda()}
    uc = {"crossattn": randn((1, 77, 2048), 203).cuda(), "vector": randn((1, 2816), 204).cuda()}
    outs = {}
    for dt in ("fp8", "bf16"):
        m = _engine(dt, tiled)
        if dt == "fp8":
            m.model.fp8_attention = True
        monkeypatch.setattr(torch, "randn_like", _SeededNoise(5000))
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            outs[dt] = m.batchify_sample(img, num_steps=3, restoration_scale=4.0, s_churn=5, s_noise=1.01, cfg_scale=4.0, seed=1234,
                                         control_scale=0.9, use_linear_CFG=True, cfg_scale_start=1.0, c=c, uc=uc).float().cpu()
        if dt == "fp8":
            assert not [str(r.message) for r in rec], [str(r.message) for r in rec]
            assert m.model.diffusion_model._fp8_attention and m.model.control_model._fp8_attention
        del m
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs["fp8"]).all())
    e = _rel(outs["fp8"], outs["bf16"])
    print(f"engine ({'tiled' if tiled else 'untiled'}) fp8 linears + attention vs bf16: rel_fro={e:.4g}")
    assert e <= ENGINE_BOUND


def test_sharded_fp8_attention_bit_identical_to_single_gpu():
    import json
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(root, "tools", "check_multigpu.py"), "--fp8-attention"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert res["dtype"] == "fp8" and res["fp8_attention"] and res["finite"] and res["sampler_sharded_equals_single"]
    assert res["identical_on_all_ranks"]
