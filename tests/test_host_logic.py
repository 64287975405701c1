"""CPU tests: C-ABI library loads and exports every declared symbol; host-side integer bookkeeping and float32 schedule
of the product (supir_b200) equal the reference's golden values; the product refuses to run without CUDA."""
import json
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(os.path.dirname(__file__), "golden")


def bits(t):
    return np.asarray(t, dtype=np.float32).view(np.uint32).tolist()


@pytest.fixture(scope="module")
def book():
    with open(os.path.join(G, "bookkeeping.json")) as f:
        return json.load(f)


def test_library_loads_and_exports_every_declared_symbol():
    from supir_b200 import _native
    lib = _native.load()
    header = open(os.path.join(ROOT, "include", "supir_b200.h")).read()
    declared = set(re.findall(r"\b(supir_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 35
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/supir_b200.h but not exported"
    assert declared == set(_native.EXPORTED_SYMBOLS), declared ^ set(_native.EXPORTED_SYMBOLS)
    assert lib.supir_version() >= 100
    assert lib.supir_last_error() is not None


def test_text_conditioner_entry_points_reject_bad_arguments_before_any_launch():
    """Argument validation of the textenc.cu entry points (no GPU needed: they return before touching the device) — the error
    convention of the boundary: negative return code + supir_last_error(), turned into SupirNativeError by the binding."""
    import ctypes
    from supir_b200 import _native
    lib = _native.load()
    p = ctypes.c_void_p(64)            # a non-null, aligned dummy pointer; never dereferenced on these paths
    cases = [("supir_attention_small_bf16", (p, 768, p, 768, p, 768, p, 768, 2, 12, 77, 32, 0.125, 1, None), "head_dim"),
             ("supir_attention_small_bf16", (p, 768, p, 768, p, 768, p, 768, 2, 12, 200, 64, 0.125, 1, None), "tokens"),
             ("supir_activation_bf16", (p, 64, p, 64, 4, 64, 7, None), "mode"),
             ("supir_gather_rows_f32", (p, 6, 10, p, None, 0, 0, p, 6, 4, 6, None), "multiples of 4"),
             ("supir_layernorm_f32", (p, 64, None, 0, None, 0, 4, 64, p, p, 1e-5, None), "bad args")]
    for name, args, needle in cases:
        assert getattr(lib, name)(*args) < 0, name
        assert needle in lib.supir_last_error().decode(), (name, lib.supir_last_error())
        with pytest.raises(_native.SupirNativeError):
            _native.call(name, *args)
    from supir_b200 import ops
    with pytest.raises(_native.SupirNativeError):
        ops.attention_small(*(torch.zeros(77, 64, dtype=torch.bfloat16),) * 4, 1, 1, 77)      # CPU tensors: no fallback


def test_attention_entry_points_reject_bad_arguments_before_any_launch():
    """Argument validation of the attention.cu entry points: the final store writes two 16-bit outputs as one 32-bit word, so
    `out` must be 4-byte aligned, and at head_dim 64 every leading dimension must cover the H * 64 columns (a shorter ldo
    would let the last row write past the buffer). Both are rejected before any tensor map is encoded or anything launched."""
    import ctypes
    from supir_b200 import _native
    lib = _native.load()
    p = ctypes.c_void_p(64)            # a non-null, aligned dummy pointer; never dereferenced on these paths
    odd = ctypes.c_void_p(66)          # 2-byte aligned: a bf16 view that starts at an odd column
    h64 = lambda out, ldq, ldk, ldv, ldo: (p, ldq, p, ldk, p, ldv, out, ldo, 2, 5, 77, 77, 64, 0.125, None)  # noqa: E731
    cases = []
    for name in ("supir_attention_bf16", "supir_attention_f16"):
        cases += [(name, h64(odd, 320, 320, 320, 320), "4-byte aligned"),
                  (name, h64(p, 256, 320, 320, 320), ">= H * 64"),
                  (name, h64(p, 320, 256, 320, 320), ">= H * 64"),
                  (name, h64(p, 320, 320, 256, 320), ">= H * 64"),
                  (name, h64(p, 320, 320, 320, 312), ">= H * 64")]
    cases.append(("supir_attention_1head_bf16", (p, 512, p, 512, p, 512, odd, 512, 1, 100, 512, 0.04, None), "4-byte aligned"))
    for name, args, needle in cases:
        assert getattr(lib, name)(*args) < 0, name
        assert needle in lib.supir_last_error().decode(), (name, lib.supir_last_error())
        with pytest.raises(_native.SupirNativeError):
            _native.call(name, *args)


def test_no_cpu_fallback():
    from supir_b200 import _native, ops
    with pytest.raises(_native.SupirNativeError):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    from supir_b200 import vae
    with torch.device("meta"):
        pass
    enc_cfg = dict(ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[], in_channels=3, resolution=32, z_channels=4)
    with pytest.raises(RuntimeError):
        vae.Encoder(**enc_cfg)(torch.zeros(1, 3, 16, 16))


def test_product_windows_tiles_and_schedule_match_reference(book):
    from supir_b200 import denoiser as dn, sampling, vae
    for case in book["sliding_windows"]:
        assert [list(c) for c in sampling._sliding_windows(*case["args"])] == case["windows"]
    for case, crop in zip(book["split_tiles"], book["crop"]):
        h, w, tile, dec = case["args"]
        ib, ob = vae.split_tiles(h, w, tile, dec)
        assert ib == case["in"] and ob == case["out"]
        for i, o, ref in zip(ib, ob, crop["crops"]):
            th, tw = (i[3] - i[2]), (i[1] - i[0])
            th, tw = (th * 8, tw * 8) if dec else (th // 8, tw // 8)
            y0, y1, x0, x1 = vae.crop_margins(th, tw, i, o, dec)
            idx = torch.arange(th * tw).view(th, tw)[y0:y1, x0:x1]
            assert [int(idx[0, 0]), int(idx[-1, -1]), idx.shape[0], idx.shape[1]] == ref
    for lb, ub, ref in book["best_tile"]:
        assert vae.get_best_tile_size(lb, ub) == ref
    disc = dn.LegacyDDPMDiscretization()
    for n, ref in book["sigmas"].items():
        assert bits(disc(int(n)).numpy()) == ref
    den = dn.DiscreteDenoiserWithControl(
        weighting_config={"target": "sgm.modules.diffusionmodules.denoiser_weighting.EpsWeighting"},
        scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"}, num_idx=1000,
        discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"})
    assert bits(den.sigmas.numpy()) == book["denoiser_table"]
    probe = np.array(book["sigma_to_idx"]["sigma"], dtype=np.uint32).view(np.float32)
    assert [den.quantize_host(float(s))[1] for s in probe] == book["sigma_to_idx"]["idx"]
    assert den.sigma_to_idx(torch.tensor(probe)).tolist() == book["sigma_to_idx"]["idx"]
    g = np.load(os.path.join(G, "gaussian_weights.npz"))
    assert np.array_equal(sampling.gaussian_weights(128, 128, 1, device="cpu").numpy(), g["w128"])
    assert np.array_equal(sampling.gaussian_weights(16, 24, 2, device="cpu").numpy(), g["w16x24"])


def test_denoiser_host_table_follows_a_loaded_sigma_buffer():
    """`denoiser.sigmas` is a persistent buffer of the reference class (denoiser.py:43): a checkpoint's table replaces the
    constructed one there, so the host-side copy the fused sampler path quantises against has to follow it."""
    from supir_b200 import denoiser as dn
    den = dn.DiscreteDenoiserWithControl(
        weighting_config={"target": "sgm.modules.diffusionmodules.denoiser_weighting.EpsWeighting"},
        scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"}, num_idx=1000,
        discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"})
    sq, idx = den.quantize_host(3.0)
    assert abs(sq - 3.0) < 0.01 and int(den.sigma_to_idx(torch.tensor([3.0]))[0]) == idx
    den.load_state_dict({"sigmas": den.sigmas * 2})
    sq2, idx2 = den.quantize_host(3.0)
    assert idx2 != idx and abs(sq2 - 3.0) < 0.02 and int(den.sigma_to_idx(torch.tensor([3.0]))[0]) == idx2


def test_step_constants_match_oracle_arithmetic():
    """The host-side float32 scalars of a step equal what the oracle computes with float32 tensors."""
    from oracle import sampler as osamp
    from supir_b200 import sampling
    guider = {"target": "sgm.modules.diffusionmodules.guiders.LinearCFG", "params": {"scale": 1.0, "scale_min": 4.0}}
    smp = sampling.RestoreEDMSampler(num_steps=50, restore_cfg=4.0, s_churn=5, s_noise=1.01, guider_config=guider,
                                     discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"})
    sig = smp.host_sigmas()
    ref = osamp.legacy_ddpm_sigmas(50)
    assert bits(sig) == bits(ref.numpy())
    for i in (0, 1, 17, 48, 49):
        k = smp.step_constants(sig, i, 0.9, True, 0.2)
        s, ns = ref[i:i + 1], ref[i + 1:i + 2]
        gamma = min(5 / 50, 2 ** 0.5 - 1)
        sh = s * (gamma + 1.0)
        assert np.float32(k["sigma_hat"]) == sh.numpy()[0]
        assert np.float32(k["dt"]) == (ns - sh).numpy()[0]
        nm = (1.01 * ((sh ** 2 - s ** 2) ** 0.5)).numpy()[0]
        assert abs(k["noise_mul"] - nm) <= 1e-6 * nm
        assert k["use_restore"] == bool(ns[0] > 0.05)
        if k["use_restore"]:
            assert abs(k["restore_mul"] - float((s / 14.6146) ** 4.0)) <= 1e-6
        assert abs(smp.guider.scale_host(k["sigma_hat"]) - float(osamp.linear_cfg_scale(1.0, 4.0, sh)[0])) <= 1e-6
        assert abs(k["control_scale"] - ((float(s[0]) / 14.6146) * (0.2 - 0.9) + 0.9)) <= 1e-7


def test_shard_windows_partition():
    from supir_b200.sampling import shard_windows
    for nw in (1, 7, 49, 64, 225):
        for world in (1, 2, 4, 8):
            seen = []
            for r in range(world):
                per, lo, hi = shard_windows(nw, world, r)
                assert 0 <= lo <= hi <= nw and hi - lo <= per
                seen += list(range(lo, hi))
            assert seen == list(range(nw))          # contiguous, ordered, complete


def test_state_dict_keys_match_reference_fixture():
    """Key names/shapes of the product's modules equal the reference's (fixtures were dumped from the reference)."""
    from supir_b200 import nets, vae, wrappers
    g = np.load(os.path.join(G, "unet_fullwidth_depth1.npz"))
    cfg, shapes = json.loads(str(g["cfg"])), json.loads(str(g["shapes"]))
    with torch.device("meta"):
        w = wrappers.ControlWrapper(nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **cfg))
        w.load_control_model(nets.GLVControl(input_upscale=1, **cfg))
    assert {k: list(v.shape) for k, v in w.state_dict().items()} == shapes
    g = np.load(os.path.join(G, "vae_tiny.npz"))
    with torch.device("meta"):
        ae = vae.AutoencoderKLInferenceWrapper(embed_dim=4, ddconfig=json.loads(str(g["cfg"])), lossconfig={"target": "torch.nn.Identity"})
    assert {k: list(v.shape) for k, v in ae.state_dict().items()} == json.loads(str(g["shapes"]))


def test_config_factory_resolves_reference_targets():
    from supir_b200 import config
    cfg = config.load_yaml(os.path.join(ROOT, "tests", "golden", "SUPIR_v0_tiled_sampler.yaml"))
    smp = config.instantiate_from_config(dict(cfg["sampler_config"], params=dict(cfg["sampler_config"]["params"], device="cpu")))
    assert type(smp).__name__ == "TiledRestoreEDMSampler" and type(smp).__module__ == "supir_b200.sampling"
    assert smp.tile_size == 128 and smp.tile_stride == 64 and type(smp.guider).__name__ == "LinearCFG"


def test_vae_step_fusion_plan():
    """Host-side step list of the VAE nets (vae._VAENet.pack / _fused_steps): every SiLU is folded into the GroupNorm before
    it and every skip-connection add into the conv / attention before it, so no standalone 'silu' or 'add_res' step runs."""
    from supir_b200 import vae
    cfg = dict(ch=32, out_ch=3, ch_mult=(1, 2), num_res_blocks=1, attn_resolutions=[], in_channels=3, resolution=32, z_channels=4)
    for net in (vae.Encoder(double_z=True, **cfg), vae.Decoder(**cfg)):
        net.pack()
        raw = [s[0] for s in net._steps]
        fused = net._fused_steps()
        kinds = [s[0] for s, _ in fused]
        assert "silu" not in kinds and "add_res" not in kinds
        assert raw.count("silu") == sum(1 for s, f in fused if s[0] == "norm" and f)
        assert raw.count("add_res") == sum(1 for s, f in fused if s[0] in ("conv", "attn") and f)
        # every skip that is stored is consumed by exactly one fused add
        assert raw.count("store_res") == raw.count("add_res")


def test_entry_exit_conv_weight_packing():
    """Tensor-core operands of the Cin<=8 / Cout<=8 convs: k = ci*9 + tap for the im2col GEMM, (kh, kw, cin) rows padded to
    8 output channels for the implicit-GEMM conv; padding is zero so the extra columns / rows cannot leak into the result."""
    from supir_b200 import ops
    w = torch.randn(16, 4, 3, 3)
    wp = ops.pack_small_cin_weight(w)
    assert wp.shape == (16, 64) and wp.dtype == torch.bfloat16
    assert torch.equal(wp[:, :36].float(), w.reshape(16, 36).to(torch.bfloat16).float()) and float(wp[:, 36:].abs().max()) == 0.0
    assert ops.pack_small_cin_weight(torch.randn(8, 8, 3, 3)).shape == (8, 128)          # 72 taps -> two 64-column k-blocks
    wc, bc = torch.randn(3, 16, 3, 3), torch.randn(3)
    p, b8 = ops.pack_small_cout_weight(wc, bc)
    assert p.shape == (8, 144) and b8.shape == (8,)
    assert torch.equal(p[:3].float(), wc.permute(0, 2, 3, 1).reshape(3, -1).to(torch.bfloat16).float())
    assert float(p[3:].abs().max()) == 0.0 and float(b8[3:].abs().max()) == 0.0
    assert torch.equal(b8[:3], bc.to(torch.bfloat16).float())


def test_bench_clock_sampler_windows():
    """bench.ClockSampler reports the samples of the timed region, or, when the region was shorter than nvidia-smi's period,
    the last samples of the warm-up + timed load, and says which."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    class _P:
        def terminate(self):
            pass
    c = bench.ClockSampler(0)
    c.proc = _P()
    c.lines = ["1500, 1965, 900.1, Not Active, Not Active, Not Active, Active"] * 3
    c.mark()
    r = c.stop()
    assert r["sm_mhz"] == 1500.0 and r["reasons"] == ["sw_power_cap"] and r["window"].startswith("warm-up")
    c.lines.append("1600, 1965, 910.0, Not Active, Not Active, Not Active, Not Active")
    r = c.stop()
    assert r["sm_mhz"] == 1600.0 and r["samples"] == 1 and r["window"] == "timed region" and r["reasons"] == []
    assert bench.ClockSampler(0).stop()["sm_mhz"] is None
