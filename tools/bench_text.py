"""Text-tower encode time on the engine, in one call on one GPU: 80 sequences of 77 tokens (the size of an 80-prompt
batch) through the 512 x 12 tower (ViT-B/32, ViT-B/16, every SLIP model) and the 768 x 12 tower (ViT-L/14), seeded
synthetic weights, on the fused causal attention and on the batched-GEMM chain (PXR_FUSED_ATTN=0).  Host clock around
pxr_encode_text, which ends in a stream synchronise; the median of `reps` calls after two warm-up calls.  Also the GPU's
name and power limit.  Prints one JSON line; writes nothing.

    python tools/bench_text.py [reps]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402
from pixray_b200 import tokenizer as TK  # noqa: E402


def gpu_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # noqa: BLE001
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rng = np.random.default_rng(0)
    ids = np.zeros((80, 77), dtype=np.int32)
    for b in range(80):
        L = int(rng.integers(3, 20))
        ids[b, :L + 2] = [TK.SOT] + list(rng.integers(1, TK.SOT, L)) + [TK.EOT]
    res = gpu_info()
    for width in (512, 768):
        sd = {**S.clip_state_dict(dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=width), 1),
              **S.clip_text_state_dict(width, 12, width, 2)}
        for fused in (1, 0):
            os.environ["PXR_FUSED_ATTN"] = str(fused)
            eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(8, 8), cutn=2,
                               clip=[dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=width)])
            eng.load_module(E.MOD_CLIP0, sd)
            eng.finalize()
            for _ in range(2):
                eng.encode_text(0, ids)
            times = []
            for _ in range(reps):
                t0 = time.perf_counter()
                eng.encode_text(0, ids)
                times.append(time.perf_counter() - t0)
            res[f"w{width}_{'fused' if fused else 'chain'}_ms_per_80"] = round(1e3 * float(np.median(times)), 3)
            eng.close()
    os.environ.pop("PXR_FUSED_ATTN", None)
    res["power_limit_read_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
