"""Oracle for perceptors of different input resolutions: one ascend_txt + backward over a cutoutsTable
(pixray.py:642-649, 1243-1406), built from oracle/ref_path.py's make_cutouts / encode_image / prompt_loss and one autograd
graph.  tests/golden/multires_ascend.npz (oracle/make_golden_multires.py, the unmodified reference) pins it.
"""
import torch

from oracle import ref_path as R


def iterate_sets(out, sets, perceptors, prompts, image_prompts=(), aux=(), zoom_padding="border", fill=0.0, aspect=1.0,
                 synth_fn=None):
    """out: image [1, 3, H, W] (or z when synth_fn is given: out = synth_fn(z), and z_grad is returned too).
    sets: the cutoutsTable in its order, dicts(cs, transforms [cutn, 3, 3], noise_facs, noise, jitter) -- every entry
    cut from the same image with its own cached transforms (pixray.py:1266-1268), sharing the padding mode and fill.
    perceptors: (model with encode_image, index of its set); prompts: per perceptor (embed [n, D], weight, stop) rows.
    image_prompts: (target image, weight), cut per perceptor with its own set's cached transforms and noise, no
    ColorJitter (pixray.py:1308-1336), scored after its text prompts.  aux: (weight, kind, fn): kind "cutouts" gives one
    entry per set, fn(batch) in set order (SaturationLoss / PaletteLoss / SmoothnessLoss return such lists); "image"
    one entry fn(out, embeds of the last perceptor).  Returns dict(losses, image_grad, z_grad, batches, embeds)."""
    z = None
    if synth_fn is not None:
        z = out.detach().clone().requires_grad_(True)
        out = synth_fn(z)
    else:
        out = out.detach().clone().requires_grad_(True)
    out.retain_grad()

    def cut(img, s, jitter=True):
        return R.make_cutouts(img, s["transforms"], s["cs"], zoom_padding, fill, s.get("noise_facs"), s.get("noise"),
                              jitter=s.get("jitter") if jitter else None, aspect=aspect)

    batches = [cut(out, s) for s in sets]
    losses, embeds = [], []
    for (model, si), pms in zip(perceptors, prompts):
        iii = R.encode_image(model, batches[si])
        embeds.append(iii)
        for (embed, weight, stop) in pms:
            losses.append(R.prompt_loss(iii, embed, weight, stop))
        for (timg, weight) in image_prompts:
            with torch.no_grad():
                te = R.encode_image(model, cut(timg.to(out.dtype), sets[si], jitter=False))
            losses.append(R.prompt_loss(iii, te, weight, float("-inf")))
    for (weight, kind, fn) in aux:
        if kind == "cutouts":
            losses += [weight * fn(b) for b in batches]
        else:
            losses.append(weight * fn(out, embeds[-1]))
    sum(losses).backward()
    return dict(losses=[l.detach() for l in losses], image_grad=out.grad.detach(),
                z_grad=None if z is None else z.grad.detach(), batches=[b.detach() for b in batches],
                embeds=[e.detach() for e in embeds])
