"""taming's GumbelVQ, the VQGAN of pixray's openimages_f16_8192 (vqgan.py:124-131), restated for the oracle: the VQModel of
ref_path.py with GumbelQuantize in place of VectorQuantizer.  The decoder, post_quant_conv, encoder and quant_conv are
ref_path's; the quantiser keeps its codebook as quantize.embed and adds quantize.proj, a 1x1 convolution from
z_channels to n_embed logits.

GumbelQuantize.forward in eval mode [UPSTREAM taming/modules/vqvae/quantize.py, un-vendored]: hard = True, so
F.gumbel_softmax(logits, tau, dim=1, hard=True) is the one-hot of argmax(logits + g) made straight-through,
y_hard - y_soft.detach() + y_soft, and z_q = einsum('b n h w, n d -> b d h w', that, embed.weight).  g is torch's
-log(Exp(1)) noise; here it is an argument, so the engine and the oracle can be handed the same draw."""
import torch
from torch import nn
from torch.nn import functional as F

from . import ref_path as R


class GumbelVQModel(R.VQModel):
    """ref_path.VQModel with the GumbelVQ key layout: quantize.embed [n_embed, embed_dim] and, with the encoder,
    quantize.proj [n_embed, z_channels, 1, 1]."""

    def __init__(self, n_embed=8192, embed_dim=256, with_encoder=False, **dd):
        super().__init__(n_embed=n_embed, embed_dim=embed_dim, with_encoder=with_encoder, **dd)
        self.quantize = nn.Module()
        self.quantize.embed = nn.Embedding(n_embed, embed_dim)
        if with_encoder:
            self.quantize.proj = nn.Conv2d(dd.get("z_channels", 256), n_embed, 1)

    @property
    def codebook(self):
        return self.quantize.embed.weight

    def encode(self, x, noise, tau=1.0):
        """VQModel.encode of a GumbelVQ: quantize(quant_conv(encoder(x))) with the Gumbel draws `noise` [B, n_embed, h, w]
        -> (z_q [B, C, h, w], indices [B * h * w], pre-quantisation h, logits)."""
        h = self.quant_conv(self.encoder(x))
        z_q, idx, logits = gumbel_quantize(h, self.quantize.proj.weight, self.quantize.proj.bias, self.codebook, noise, tau)
        return z_q, idx, h, logits


def gumbel_quantize(h, proj_weight, proj_bias, embed, noise, tau=1.0):
    """GumbelQuantize.forward, eval mode (hard), with the Gumbel noise given: -> (z_q, indices [B * h * w], logits)."""
    logits = F.conv2d(h, proj_weight, proj_bias)
    y_soft = ((logits + noise) / tau).softmax(dim=1)
    idx = y_soft.max(dim=1)[1]  # F.gumbel_softmax's own arg-max
    y_hard = torch.zeros_like(logits).scatter_(1, idx[:, None], 1.0)
    one_hot = y_hard - y_soft.detach() + y_soft
    z_q = torch.einsum("bnhw,nd->bdhw", one_hot, embed)
    return z_q, idx.reshape(-1), logits


def vqgan_synth(model, z):
    """VqganDrawer.synth of a GumbelVQ (vqgan.py:190-193): the nearest code of quantize.embed, then the decoder."""
    zq, _ = R.vector_quantize(z.movedim(1, 3), model.codebook)
    return R.clamp_with_grad(model.decode(zq.movedim(3, 1)).add(1).div(2), 0, 1)
