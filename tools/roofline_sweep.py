"""BASELINE config 5: roofline sweep 256^2 -> 1024^2, 16 -> 128 samples/ray, translucent / opaque scene, at 1 GPU or -- under
torchrun -- frame-sharded over N GPUs with the uint8 all-gather at the end of every clip (weak scaling: T frames per rank).

    python tools/roofline_sweep.py [precision]                                                     # 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/roofline_sweep.py fp16

Rank 0 prints one JSON line per configuration: aggregate fps (device time, max over ranks), valid samples S per frame, head-kernel
ms/frame (CUDA events inside libgfpp, rank 0), achieved algorithmic GB/s and its fraction of the measured HBM peak (SURVEY 8(d)),
the fraction of the L2 scattered-sector ceiling (1 sector / clk / SM) and the tensor fraction (algorithmic MLP flops / measured
sustained dense bf16 peak)."""
import ctypes
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from genefaceplusplus_b200 import _capi, scene as scn  # noqa: E402
from genefaceplusplus_b200 import dist as gdist  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorso  # noqa: E402

prec = sys.argv[1] if len(sys.argv) > 1 else "fp16"
world = int(os.environ.get("WORLD_SIZE", "1")); rank = int(os.environ.get("RANK", "0")); local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
peak, bf16 = pk.get("hbm_gbs", 3350.0), pk.get("bf16_tflops_sustained", 989.0)
n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
sectors_per_sample = 2 * 16 * (1 if prec in ("fp16", "robust") else 2)
L = _capi.lib()
L.gfpp_profile_enable(1)
for size in (256, 512, 1024):
    for ms in (16, 32, 64, 128):
        for ds in (1.0, 64.0):
            T = 16 if size < 1024 else 8                       # frames per rank
            sc = scn.Scene(H=size, W=size, T=T * world, torso=True, max_steps=ms, density_scale=ds)
            m = RADNeRFTorso(sc.hparams); m.load_state_dict(sc.state); m.density_scale = ds; m.mlp_precision = prec
            m = m.to(dev).eval()
            s, e = gdist.frame_block(T * world, rank, world)
            poses = torch.stack([sc.pose(t) for t in range(s, e)]).to(dev)
            feat = m.cal_cond_feat_clip(sc.cond.to(dev))[s:e]
            pose6 = scn.convert_poses(poses.cpu()).to(dev)
            u8 = torch.empty(T, size * size, 3, dtype=torch.uint8, device=dev)
            kw = dict(poses_c2w=poses, intrinsics=sc.intrinsics, H=size, W=size, pose6=pose6, bg_coords=sc.bg_coords.to(dev), bg_color=sc.bg_color.to(dev),
                      dt_gamma=sc.hparams["dt_gamma"], max_steps=ms, T_thresh=0.01, want_torso_maps=False, want_stats=True, want_aux=False, u8_out=u8)

            def clip():
                res = m.render_frames(feat, **kw)
                if world > 1:
                    gdist.gather_frames(u8, T * world)
                return res

            for _ in range(3):
                res = clip()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                res = clip()
            e1.record(); torch.cuda.synchronize()
            tms = torch.tensor([e0.elapsed_time(e1)], device=dev)
            if world > 1:
                dist.all_reduce(tms, op=dist.ReduceOp.MAX)
            buf = (ctypes.c_float * 4)(); L.gfpp_profile_read(buf)
            st = res["stats"].cpu()
            S = st[:, 2].float().mean().item(); N = size * size
            head = buf[0] / 1000.0 / T
            bytes_ = S * 2048 + N * 20
            if rank == 0:
                print(json.dumps({"n_gpus": world, "size": size, "max_steps": ms, "density_scale": ds, "precision": prec,
                                  "fps": world * 3 * T / (tms.item() / 1000.0), "frames_per_gpu": T,
                                  "S_per_frame": S, "B_total": int(st[0, 0]), "head_ms_per_frame": head * 1000, "achieved_GBps": bytes_ / head / 1e9,
                                  "hbm_frac": bytes_ / head / 1e9 / peak, "fp32_equiv_TFLOPs": S * 178944 / head / 1e12,
                                  "tensor_frac": S * 178944 / head / 1e12 / bf16,
                                  "l2_sector_frac": S * sectors_per_sample / head / (n_sm * 1.965e9)}), flush=True)
            del m
            torch.cuda.empty_cache()
if world > 1:
    dist.destroy_process_group()
