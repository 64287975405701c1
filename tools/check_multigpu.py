"""torchrun --nproc-per-node N tools/check_multigpu.py [--dtype bf16|fp16|fp8] [--fp8-convs] [--fp8-attention] : the unit-sharded tiled sampler and the
tile-sharded VAE give the same result as the single-GPU path, bit for bit, on every rank (also run by tests/test_gpu_multigpu.py and,
with --dtype fp16 / fp8 / --fp8-convs, by tests/test_gpu_fp16.py / test_gpu_fp8.py / test_gpu_fp8_conv.py when >= 2 GPUs). --dtype
is the compute dtype of the diffusion networks; --fp8-convs (implies --dtype fp8) also runs the ResBlocks' 3x3 convolutions in FP8,
--fp8-attention (implies --dtype fp8) the self-attentions and ZeroCrossAttn."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist
from weights import make_state_dict, randn

def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from supir_b200 import denoiser as dn, nets, sampling, vae, wrappers
    g = np.load(os.path.join(ROOT, "tests", "golden", "unet_fullwidth_depth1.npz"))
    cfg = json.loads(str(g["cfg"]))
    sd = make_state_dict(json.loads(str(g["shapes"])), seed=31)
    with torch.device("meta"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **cfg)
        ctrl = nets.GLVControl(input_upscale=1, **cfg)
    fp8_convs, fp8_attention = "--fp8-convs" in sys.argv, "--fp8-attention" in sys.argv
    dname = sys.argv[sys.argv.index("--dtype") + 1] if "--dtype" in sys.argv else ("fp8" if fp8_convs or fp8_attention else "bf16")
    net = wrappers.ControlWrapper(unet, dtype={"bf16": torch.bfloat16, "fp16": torch.float16, "fp8": torch.float8_e4m3fn}[dname])
    net.fp8_convs, net.fp8_attention = fp8_convs, fp8_attention
    net.load_control_model(ctrl)
    net.to_empty(device="cuda")
    net.load_state_dict(sd)
    disc = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
    den = dn.DiscreteDenoiserWithControl(weighting_config={"target": "sgm.modules.diffusionmodules.denoiser_weighting.EpsWeighting"},
                                         scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
                                         num_idx=1000, discretization_config=disc).cuda()
    denoiser = sampling.FusedDenoiser(den, net)
    def run(shard):
        smp = sampling.TiledRestoreEDMSampler(tile_size=32, tile_stride=16, tile_batch=3, num_steps=3, restore_cfg=4.0, s_churn=5,
                                              s_noise=1.01, discretization_config=disc,
                                              guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearCFG", "params": {"scale": 1.0, "scale_min": 4.0}})
        smp.shard = shard
        torch.manual_seed(7)
        x = randn((1, 4, 80, 64), 1).cuda()
        c = {"control": randn((1, 4, 80, 64), 2).cuda(), "crossattn": randn((1, 77, 2048), 3).cuda(), "vector": randn((1, 2816), 4).cuda()}
        uc = {"control": c["control"], "crossattn": randn((1, 77, 2048), 5).cuda(), "vector": randn((1, 2816), 6).cuda()}
        return smp(denoiser, x, cond=c, uc=uc, x_center=randn((1, 4, 80, 64), 7).cuda(), control_scale=0.9)
    a = run(True)
    b = run(False)
    same = torch.equal(a, b)

    def run_untiled(shard):      # CFG-branch parallelism of the untiled sampler (ranks 0 / 1 carry one branch each)
        smp = sampling.RestoreEDMSampler(num_steps=3, restore_cfg=4.0, s_churn=5, s_noise=1.01, discretization_config=disc,
                                         guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearCFG", "params": {"scale": 1.0, "scale_min": 4.0}})
        smp.shard = shard
        torch.manual_seed(9)
        x = randn((1, 4, 48, 40), 11).cuda()
        c = {"control": randn((1, 4, 48, 40), 12).cuda(), "crossattn": randn((1, 77, 2048), 13).cuda(), "vector": randn((1, 2816), 14).cuda()}
        uc = {"control": c["control"], "crossattn": randn((1, 77, 2048), 15).cuda(), "vector": randn((1, 2816), 16).cuda()}
        return smp(denoiser, x, cond=c, uc=uc, x_center=randn((1, 4, 48, 40), 17).cuda(), control_scale=0.9)
    pair_same = torch.equal(run_untiled(True), run_untiled(False))
    gathered = [torch.empty_like(a) for _ in range(world)]
    dist.all_gather(gathered, a)
    same_ranks = all(torch.equal(gathered[0], t) for t in gathered)
    # tiled VAE
    gv = np.load(os.path.join(ROOT, "tests", "golden", "vae_tiny.npz"))
    with torch.device("cuda"):
        ae = vae.AutoencoderKLInferenceWrapper(embed_dim=4, ddconfig=json.loads(str(gv["cfg"])), lossconfig={"target": "torch.nn.Identity"})
    ae.load_state_dict(make_state_dict(json.loads(str(gv["shapes"])), seed=71))
    zbig = randn((1, 4, 40, 52), 84).cuda()
    d_sharded = ae.decoder.tiled_forward(zbig, 16, shard=True)
    d_single = ae.decoder.tiled_forward(zbig, 16, shard=False)
    vae_same = torch.equal(d_sharded, d_single)
    ref = torch.from_numpy(gv["dec_tiled"]).cuda()
    rel = float((d_sharded - ref).norm() / ref.norm())
    if rank == 0:
        print(json.dumps({"world": world, "dtype": dname, "fp8_convs": fp8_convs, "fp8_attention": fp8_attention, "sampler_sharded_equals_single": same, "untiled_branch_parallel_equals_single": pair_same, "identical_on_all_ranks": same_ranks,
                          "vae_sharded_rel_fro_vs_reference": rel, "vae_sharded_equals_single": vae_same, "finite": bool(torch.isfinite(a).all())}))
    dist.barrier()
    dist.destroy_process_group()
    assert same and pair_same and same_ranks and vae_same and rel < 3e-2

main()
