"""Generate tests/golden/slip_perceptor.npz by running the UNMODIFIED reference slip.py SLIP_Base (container-only).

    python -m oracle.make_golden_slip

SLIP_Base (slip.py:84-157) loads `models/slip_base_100ep.pt` from the working directory, strips the checkpoint's
`module.` prefix, builds SLIP/models.py's SLIP_VITB16 and runs its preprocess / encode_image.  Its third-party leaves
are absent here and come in as stub modules:
  * timm: registry.register_model, create_model (-> oracle/slip_ref.py's restatement of timm 0.5's VisionTransformer, with
    TWO blocks instead of twelve so the checkpoint stays small) and models.vision_transformer._create_vision_transformer;
  * clip.clip, ftfy (imported by SLIP's tokenizer), util.wget_file (never called: the checkpoint exists);
  * Tensor.cuda / Module.cuda are the identity (slip.py:139, 166 run on this CPU-only container), as make_golden_aux.py
    does for EdgeLoss; torch.load's weights_only mode is told about argparse.Namespace, the checkpoint's `args`.
The checkpoint is written into a scratch working directory: the whole SLIP model seeded, then its image tower replaced by
pixray_b200.synthetic.slip_state_dict(ARCH, SEED), which the test regenerates.  The golden holds the preprocessed input,
the unit embeddings and d(loss)/d(input) through encode_image for loss = sum(embeddings * DIR).
"""
import argparse
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch
from torch import nn

from oracle import slip_ref as SR
from pixray_b200 import synthetic

REFERENCE = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "slip_perceptor.npz")
ARCH = dict(width=768, layers=2, heads=12, patch=16, image_res=224, out_dim=512)
SEED = 11


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _install_stubs():
    def create_model(name, num_classes=0, **kw):
        assert name == "vit_base_patch16_224" and num_classes == 0, name
        return SR.VisionTransformer(224, 16, ARCH["width"], ARCH["layers"], ARCH["heads"])

    timm = _mod("timm", create_model=create_model)
    timm.models = _mod("timm.models")
    timm.models.registry = _mod("timm.models.registry", register_model=lambda f: f)
    timm.models.vision_transformer = _mod("timm.models.vision_transformer",
                                          _create_vision_transformer=lambda *a, **k: None)
    clip_pkg = _mod("clip")
    clip_pkg.clip = _mod("clip.clip", available_models=lambda: [], tokenize=None, load=None)
    _mod("ftfy", fix_text=lambda s: s)
    _mod("util", wget_file=lambda url, path: (_ for _ in ()).throw(RuntimeError("no network: " + url)))


def main():
    if not os.path.isdir(REFERENCE):
        raise RuntimeError("the reference checkout is only available in the authoring container")
    _install_stubs()
    torch.serialization.add_safe_globals([argparse.Namespace])
    torch.Tensor.cuda = lambda self, *a, **k: self
    nn.Module.cuda = lambda self, *a, **k: self
    spec = importlib.util.spec_from_file_location("slip", os.path.join(REFERENCE, "slip.py"))
    slip = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(slip)  # appends SLIP/ to sys.path and imports its models / tokenizer / utils

    args = argparse.Namespace(model="SLIP_VITB16", ssl_mlp_dim=64, ssl_emb_dim=32)
    torch.manual_seed(SEED)
    full = slip.models.SLIP_VITB16(rand_embed=False, ssl_mlp_dim=args.ssl_mlp_dim, ssl_emb_dim=args.ssl_emb_dim)
    sd = full.state_dict()
    sd.update(synthetic.slip_state_dict(ARCH, SEED))
    ckpt = {"state_dict": {"module." + k: v for k, v in sd.items()}, "args": args}

    g = torch.Generator().manual_seed(SEED + 1)
    # blocky cutout (8 x 8 pixel cells) in [-0.2, 1.3): compressible input, global min / max attained many times over
    imgs = torch.nn.functional.interpolate(torch.rand(1, 3, 28, 28, generator=g) * 1.5 - 0.2, scale_factor=8,
                                           mode="nearest")
    direction = torch.randn(1, ARCH["out_dim"], generator=g)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            os.makedirs("models")
            torch.save(ckpt, "models/slip_base_100ep.pt")
            perceptor = slip.SLIP_Base("SLIP_VITB16", "cpu")
            x = imgs.clone().requires_grad_(True)
            pre = perceptor.preprocess(x.detach())
            emb = perceptor.encode_image(x)
            (emb * direction).sum().backward()
        finally:
            os.chdir(cwd)
    np.savez_compressed(OUT, imgs=imgs.numpy(), preprocessed=pre.numpy(), embeds=emb.detach().numpy(),
                        direction=direction.numpy(), grad=x.grad.numpy(), seed=np.int64(SEED),
                        arch=np.array([ARCH[k] for k in ("width", "layers", "heads", "patch", "image_res", "out_dim")]))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
