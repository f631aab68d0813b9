"""BASELINE configs 3 and 5 on the GPUs the launcher gives it (informational; bench.py measures config 2, the
configuration BASELINE.json's metric is quoted on).

    python tools/bench_configs.py c3 [steps]        # vqgan 512x512, ViT-B/16 + ViT-B/32, cutn=128 (cutouts sharded over ranks)
    python tools/bench_configs.py c5 [steps]        # fft 512x512, ViT-L/14, cutn=256 (one problem per GPU: replicas)
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/bench_configs.py c3

Seeded random weights, engine-drawn cutout parameters, CUDA events on the engine stream, max over ranks."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "c3"
steps_n, warm = int(sys.argv[2]) if len(sys.argv) > 2 else 10, 3
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))

t0 = time.time()
if which == "c3":
    names, cutn, hw, shard = ["ViT-B/16", "ViT-B/32"], 128, (512, 512), world > 1
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=hw, cutn=cutn, clip=[E.CLIP_ARCH[n] for n in names], seed=0, device=local,
                       rank=rank if shard else 0, world=world if shard else 1)
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (32, 32), 3).cuda()
    workload = "vqgan 512x512, ViT-B/16 + ViT-B/32, cutn=128 (BASELINE.json configs[2])"
    lr, jobs = 0.2, 1
elif which == "c5":
    names, cutn, hw, shard = ["ViT-L/14"], 256, (512, 512), False
    eng = E.B200Engine(drawer=E.DRAWER_FFT, image_hw=hw, cutn=cutn, clip=[E.CLIP_ARCH[n] for n in names], seed=rank, device=local)
    z = (0.01 * torch.randn(eng.z_shape, device="cuda")).contiguous()
    workload = "fft 512x512, ViT-L/14, cutn=256, one prompt per GPU (BASELINE.json configs[4])"
    lr, jobs = 0.3, world
else:
    raise SystemExit("usage: bench_configs.py c3|c5 [steps]")
for i, n in enumerate(names):
    eng.load_module(E.MOD_CLIP0 + i, S.clip_state_dict(E.CLIP_ARCH[n], 1 + i))
eng.finalize()
if which == "c3" and shard:
    eng.init_comm()
for i, n in enumerate(names):
    pr = S.prompts(E.CLIP_ARCH[n]["out_dim"], (1.0, 0.1), 2 + i)
    eng.set_prompts(i, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
if rank == 0:
    print(f"setup {time.time() - t0:.1f} s", flush=True)

ext = torch.cuda.ExternalStream(eng.stream_ptr())
for it in range(warm):
    eng.iterate(z, lr, it)
eng.sync()
if world > 1:
    dist.barrier()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
w0 = time.time()
e0.record(ext)
for it in range(warm, warm + steps_n):
    eng.iterate(z, lr, it)
e1.record(ext)
eng.sync()
wall = (time.time() - w0) * 1e3
ms = e0.elapsed_time(e1)
ms = ms if ms > 0.5 * wall else wall
t = torch.tensor([ms], device="cuda", dtype=torch.float64)
if world > 1:
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
ms = float(t.item())
if rank == 0:
    flops = 2 * sum(cutn * S.vit_fwd_flops(E.CLIP_ARCH[n]) for n in names)
    if which == "c3":
        flops += 2 * S.vqgan_decoder_fwd_flops(E.VQGAN_F16_16384, hw)
    print(json.dumps({"workload": workload, "n_gpus": world, "parallelism": "cutouts sharded" if shard else f"{world} replica(s)",
                      "iters_per_sec": jobs * steps_n / (ms * 1e-3), "ms_per_step": ms / steps_n, "steps": steps_n,
                      "finite_z": bool(torch.isfinite(z).all()), "algorithmic_tflop_per_iter": flops / 1e12,
                      "whole_iter_tflops": jobs * flops * steps_n / (ms * 1e-3) / 1e12}))
if world > 1:
    dist.destroy_process_group()
