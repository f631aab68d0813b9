"""pixray's plugin surface (SURVEY.md 8b) on top of the H100 engine.

Same class / method names, argument meaning and error behaviour as the reference, so a pixray loop written against
`drawer.synth`, `MakeCutouts.__call__`, `perceptor.encode_image`, `Prompt.__call__`, `opt.step()` / `drawer.clip_z()`
runs unchanged -- each method forwards to one C entry point (include/pixray_b200.h).  Like the reference's module
globals (pixray.py:1022-1063) there is ONE session per process: the plugin objects share one `B200Engine`.

Gradients do not flow through torch autograd here: the engine owns the hand-written backward chain, so
`Session.backward()` replaces `sum(lossAll).backward()` (pixray.py:1481-1482) and writes `drawer.z.grad`.
"""
import math

import numpy as np
import torch
from torch.nn import functional as F

from . import cutouts as cut_sampler
from . import engine as E
from . import tokenizer


class DrawingInterface:
    """DrawingInterface.py:1-12 -- the declared part of the drawer contract."""

    @staticmethod
    def add_settings(parser):
        return parser

    def __init__(self, settings):
        self.settings = settings

    def load_model(self, settings, device):
        pass

    @torch.no_grad()
    def to_image(self):
        """TF.to_pil_image(self.synth(None)[0].cpu()) (vqgan.py:197-200 and the other drawers): float -> mul(255).byte()."""
        from PIL import Image
        out = self.synth(None)
        return Image.fromarray(out[0].detach().cpu().mul(255).byte().permute(1, 2, 0).numpy(), mode="RGB")


class Session:
    """The shared engine + the per-iteration state the reference keeps in globals (cur_iteration,
    global_padding_mode, global_fill_color: pixray.py:1250-1258)."""

    def __init__(self, eng: E.B200Engine):
        self.engine = eng
        self.cur_iteration = 0
        self.global_padding_mode = "reflection"
        self.global_fill_color = 0.0
        self.last_embeds = {}  # clip_idx -> the tensor Perceptor.encode_image handed out this iteration
        self.opt_kind = E.OPT_ADAM  # the engine's optimiser update rule

    def use_optimizer(self, kind):
        """A fresh optimiser of update rule `kind` (E.OPT_*) on z, as rebuild_optimisers builds one: reset_optimizer when
        the engine already runs that rule (an Adam-only session never issues anything else), set_optimizer otherwise."""
        if kind == self.opt_kind:
            self.engine.reset_optimizer()
        else:
            self.engine.set_optimizer(kind)
            self.opt_kind = kind

    def begin_iteration(self, cur_iteration, fill=None, rng=None):
        self.cur_iteration = cur_iteration
        self.global_padding_mode = "reflection" if cur_iteration % 2 == 0 else "border"  # pixray.py:1250-1253
        self.global_fill_color = float((rng or np.random).random()) if fill is None else float(fill)  # 1255-1258

    def backward(self, drawer):
        """loss.backward(): z.grad += d(sum of prompt losses)/dz (pixray.py:1481-1482)."""
        g = self.engine.backward()
        z = drawer.get_z()
        z.grad = g if z.grad is None else z.grad + g
        return g


class VqganDrawer(DrawingInterface):
    """vqgan.py:81-218 (synth 190-195, clip_z 202-204, get_z/set_z/get_z_copy 206-216)."""

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--vqgan_model", type=str, help="VQGAN model", default="imagenet_f16_16384", dest="vqgan_model")
        parser.add_argument("--vqgan_config", type=str, help="VQGAN config", default=None, dest="vqgan_config")
        parser.add_argument("--vqgan_checkpoint", type=str, help="VQGAN checkpoint", default=None, dest="vqgan_checkpoint")
        return parser

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        self.z = None

    def load_model(self, settings, device):
        self.device = device
        lo, hi = self.session.engine.z_bounds()
        self.z_min, self.z_max = lo[None, :, None, None], hi[None, :, None, None]  # vqgan.py:141-142
        # vqgan.py:124-131 (an engine class without the flag builds nearest-code VQGANs only)
        self.gumbel = getattr(self.session.engine, "gumbel", False)

    def get_opts(self, decay_divisor):
        return None  # engine builds Adam on get_z(), like pixray.py:537-539

    def get_num_resolutions(self):
        return self.session.engine.cfg.n_levels

    def init_from_tensor(self, init_tensor):
        """self.z, *_ = self.model.encode(init_tensor) (vqgan.py:174-176): taming Encoder + quant_conv + nearest code on the
        engine (pxr_vqgan_encode)."""
        self.z = self.get_z_from_tensor(init_tensor).clone()
        return self.z

    def reapply_from_tensor(self, new_tensor):
        new_z = self.get_z_from_tensor(new_tensor)
        with torch.no_grad():
            self.z.copy_(new_z)

    def get_z_from_tensor(self, ref_tensor):
        eng = self.session.engine
        if not self.gumbel:
            return eng.vqgan_encode(ref_tensor)
        # GumbelQuantize's eval forward adds F.gumbel_softmax's noise, -log(Exp(1)), to every logit: drawn here, fresh
        # for each encode, from torch's global generator, so every rank of a sharded run draws the same
        noise = -torch.empty(eng.cfg.n_embed, *eng.z_shape[2:], device=eng.device).exponential_().log()
        return eng.vqgan_encode_gumbel(ref_tensor, noise)

    def synth(self, cur_iteration):
        return self.session.engine.synth(self.z)

    def clip_z(self):
        with torch.no_grad():
            self.z.copy_(self.z.maximum(self.z_min).minimum(self.z_max))

    def get_z(self):
        return self.z

    def set_z(self, new_z):
        if self.z is None:
            self.z = new_z.detach().to(self.session.engine.device, torch.float32).contiguous().clone()
            return self.z
        with torch.no_grad():
            return self.z.copy_(new_z)

    def get_z_copy(self):
        return self.z.clone()


class FastPixelDrawer(DrawingInterface):
    """fast_pixeldrawer.py:24-110: z = colour grid, synth = nearest upsample + clamp_with_grad."""

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--pixel_size", nargs=2, type=int, help="Pixel size (width height)", default=None, dest="pixel_size")
        parser.add_argument("--pixel_scale", type=float, help="Pixel scale", default=None, dest="pixel_scale")
        return parser

    @staticmethod
    def grid_for(size, pixel_size=None, pixel_scale=None, verbose=True):
        """(num_rows, num_cols) as FastPixelDrawer.__init__ derives them (fast_pixeldrawer.py:37-63): an explicit
        pixel_size (width, height), else 40x40 on a square canvas, 40x50 on a portrait one, 80x45 on a landscape one; divided
        by pixel_scale; never larger than the canvas."""
        canvas_width, canvas_height = size
        if pixel_size is not None:
            num_cols, num_rows = pixel_size
        elif canvas_width == canvas_height:
            num_cols, num_rows = 40, 40
        elif canvas_width < canvas_height:
            num_cols, num_rows = 40, 50
        else:
            num_cols, num_rows = 80, 45
        if pixel_scale is not None and pixel_scale > 0:
            num_cols, num_rows = int(num_cols / pixel_scale), int(num_rows / pixel_scale)
        shrink = False
        if num_cols > canvas_width:
            shrink, num_cols = True, canvas_width
        if num_rows > canvas_height:
            shrink, num_rows = True, canvas_height
        if shrink and verbose:
            print("pixel grid size should not be larger than output pixel size: reducing pixel grid")
        return num_rows, num_cols

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        self.pixel_size = (session.engine.z_shape[2], session.engine.z_shape[3])
        self.output_size = session.engine.image_hw
        self.num_rows, self.num_cols = self.pixel_size
        self.z = None

    def get_opts(self, decay_divisor):
        return None

    def get_num_resolutions(self):
        return None

    def get_z_from_tensor(self, ref_tensor):
        return F.interpolate((ref_tensor + 1) / 2, size=self.pixel_size, mode="bilinear", align_corners=False)

    def init_from_tensor(self, init_tensor):
        self.z = self.get_z_from_tensor(init_tensor).to(self.session.engine.device, torch.float32).contiguous()

    def synth(self, cur_iteration):
        return self.session.engine.synth(self.z)

    def clip_z(self):
        with torch.no_grad():
            self.z.copy_(self.z.clip(0, 1))

    def get_z(self):
        return self.z

    def set_z(self, new_z):
        with torch.no_grad():
            return self.z.copy_(new_z)

    def get_z_copy(self):
        return self.z.clone()


class PixelDrawer(DrawingInterface):
    """pixeldrawer.py:110-406 for the shaped cells (pixel_type rectshift / hex / tri / diamond / knit): fixed polygons
    (pixel_shapes.py), z = their [n, 4] RGBA fill colours, rendered by the engine's polygon rasteriser
    (PXR_DRAWER_POLYGON).  The drawer owns its Adam rate, 0.03 / decay_divisor, which get_opts reports for the engine's
    fused Adam like FftDrawer does.  pixel_type rect keeps the square-grid fast path (FastPixelDrawer, chosen in
    api.do_init)."""

    @staticmethod
    def add_settings(parser):
        from .api import str2bool
        parser.add_argument("--pixel_size", nargs=2, type=int, help="Pixel size (width height)", default=None, dest="pixel_size")
        parser.add_argument("--pixel_scale", type=float, help="Pixel scale", default=None, dest="pixel_scale")
        parser.add_argument("--pixel_type", type=str, help="rect, rectshift, hex, tri, diamond, knit", default="rect", dest="pixel_type")
        parser.add_argument("--pixel_edge_check", type=str2bool, help="ensure grid is symmetric", default=True, dest="pixel_edge_check")
        parser.add_argument("--pixel_iso_check", type=str2bool, help="ensure tri and hex shapes are w/h scaled", default=True, dest="pixel_iso_check")
        return parser

    @staticmethod
    def grid_for(settings, size, verbose=True):
        """(num_rows, num_cols) of the settings on a canvas of size (width, height) (pixeldrawer.py:123-177)."""
        from . import pixel_shapes
        return pixel_shapes.grid_for(size, settings.pixel_type, getattr(settings, "pixel_size", None),
                                     getattr(settings, "pixel_scale", None), getattr(settings, "pixel_edge_check", True),
                                     getattr(settings, "pixel_iso_check", True), verbose=verbose)

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        from . import pixel_shapes
        self.session = session
        self.pixel_type = pixel_shapes.check_pixel_type(settings.pixel_type)
        self.canvas_height, self.canvas_width = session.engine.image_hw
        self.num_rows, self.num_cols = PixelDrawer.grid_for(settings, (self.canvas_width, self.canvas_height), verbose=False)
        self.z = None
        self.img = None

    def load_model(self, settings, device):
        self.device = device

    def get_opts(self, decay_divisor=1):
        return [{"lr": 0.03 / decay_divisor}]

    def get_num_resolutions(self):
        return None

    def _colours(self, tensor):
        from . import pixel_shapes
        c = pixel_shapes.init_colours(tensor, self.num_rows, self.num_cols, self.pixel_type)
        return torch.from_numpy(c).to(self.session.engine.device, torch.float32).contiguous()

    def init_from_tensor(self, init_tensor):
        """encode_image (pixeldrawer.py:200-304): every cell averages up to 4 x 4 pixels of (init_tensor + 1) / 2.  A start
        image is required: init_tensor None raises ValueError."""
        self.z = self._colours(init_tensor)

    def reapply_from_tensor(self, new_tensor):
        new_z = self._colours(new_tensor)
        with torch.no_grad():
            self.z.copy_(new_z)

    def get_z_from_tensor(self, ref_tensor):
        return None

    def synth(self, cur_iteration):
        """The render of cur_iteration's sample positions, [1, 3, H, W] (RGB: the background is transparent black)."""
        eng = self.session.engine
        eng.set_synth_iteration(cur_iteration)
        self.img = eng.synth(self.z)
        return self.img

    @torch.no_grad()
    def to_image(self):
        """The current colours rendered with the session's iteration, clipped to [0, 1] (pixeldrawer.py:369-376).  The
        reference shows its last render, which its loop refreshes every iteration through synth; here the fused iteration
        renders inside the engine, so the image is rendered afresh from the current z."""
        from PIL import Image
        img = self.synth(self.session.cur_iteration)
        arr = np.uint8(np.clip(img[0].detach().cpu().numpy().transpose(1, 2, 0), 0, 1) * 255)
        return Image.fromarray(arr, mode="RGB")

    def clip_z(self):
        with torch.no_grad():
            self.z[:, :3].clamp_(0.0, 1.0)
            self.z[:, 3].clamp_(1.0, 1.0)

    def get_z(self):
        return self.z

    def set_z(self, new_z):
        if self.z is None:
            self.z = new_z.detach().to(self.session.engine.device, torch.float32).contiguous().clone()
            return self.z
        with torch.no_grad():
            return self.z.copy_(new_z)

    def get_z_copy(self):
        return self.z.clone()


PAPER_RGBA = (242 / 255.0, 238 / 255.0, 203 / 255.0, 1.0)  # linedrawer.py:65


def line_start_points(canvas_width, canvas_height, num_paths, num_segments, rng=None):
    """The start control points of LineDrawer.load_model (linedrawer.py:73-99), [num_paths, 3 num_segments + 1, 2] float32
    canvas coordinates, drawn from `rng` (default: the `random` module, which the session seeds right before) in the
    reference's order and with its arithmetic."""
    import random
    rng = random if rng is None else rng
    bound = lambda value, low, high: max(low, min(high, value))  # noqa: E731 (linedrawer.py:23-24)
    out = []
    for _ in range(num_paths):
        points = []
        radius = 0.5
        radius_x = 0.5
        p0 = (0.5 + radius_x * (rng.random() - 0.5), 0.5 + radius * (rng.random() - 0.5))
        points.append(p0)
        for _ in range(num_segments):
            radius = 1.0 / (num_segments + 2)
            radius_x = radius * canvas_height / canvas_width
            p1 = (p0[0] + radius_x * (rng.random() - 0.5), p0[1] + radius * (rng.random() - 0.5))
            p2 = (p1[0] + radius_x * (rng.random() - 0.5), p1[1] + radius * (rng.random() - 0.5))
            p3 = (p2[0] + radius_x * (rng.random() - 0.5), p2[1] + radius * (rng.random() - 0.5))
            points += [p1, p2, p3]
            p0 = (bound(p3[0], 0, 1), bound(p3[1], 0, 1))
        points = torch.tensor(points)
        points[:, 0] *= canvas_width
        points[:, 1] *= canvas_height
        out.append(points)
    return torch.stack(out)


class LineDrawer(DrawingInterface):
    """linedrawer.py (`line_sketch`): num_paths open paths of stroke_length cubic Béziers stroked in black over paper,
    rendered and differentiated by the engine's stroke rasteriser (PXR_DRAWER_STROKES).  z is the packed
    [points | widths | paper RGBA] vector; its three Adams (get_opts) run as one fused Adam with per-range rates."""

    @staticmethod
    def add_settings(parser):
        from .api import str2bool
        parser.add_argument("--strokes", type=int, help="number strokes", default=24, dest="strokes")
        parser.add_argument("--stroke_length", type=int, help="stroke length", default=8, dest="stroke_length")
        parser.add_argument("--min_stroke_width", type=float, help="min width (percent of height)", default=0.5, dest="min_stroke_width")
        parser.add_argument("--max_stroke_width", type=float, help="max width (percent of height)", default=2, dest="max_stroke_width")
        parser.add_argument("--allow_paper_color", type=str2bool, help="allow paper color to change", default=False, dest="allow_paper_color")
        return parser

    @staticmethod
    def max_width(settings, canvas_height):
        return settings.max_stroke_width * canvas_height / 100  # linedrawer.py:52

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        self.canvas_height, self.canvas_width = session.engine.image_hw
        self.num_paths, self.stroke_length = settings.strokes, settings.stroke_length
        self.allow_paper_color = bool(settings.allow_paper_color)
        self.z = None
        self.img = None

    def load_model(self, settings, device):
        """The start geometry (linedrawer.py:44-126): points from `random`, every width max_width / 10, the paper colour."""
        self.device = device
        self.max_width = LineDrawer.max_width(settings, self.canvas_height)
        points = line_start_points(self.canvas_width, self.canvas_height, self.num_paths, self.stroke_length)
        widths = torch.full((self.num_paths,), float(torch.tensor(self.max_width / 10)))
        paper = torch.tensor(PAPER_RGBA)
        z = torch.cat([points.reshape(-1), widths, paper])
        self.z = z.to(self.session.engine.device, torch.float32).contiguous()

    def get_opts(self, decay_divisor=1):
        """The rates of the points, widths and (with allow_paper_color) paper Adams (linedrawer.py:128-136)."""
        opts = [{"lr": 1.0 / decay_divisor}, {"lr": 0.1 / decay_divisor}]
        if self.allow_paper_color:
            opts.append({"lr": 0.01 / decay_divisor})
        return opts

    def get_num_resolutions(self):
        return None

    def rand_init(self, toksX, toksY):
        pass

    def init_from_tensor(self, init_tensor):
        pass  # the reference leaves it a TODO (linedrawer.py:142-144)

    def reapply_from_tensor(self, new_tensor):
        pass

    def get_z_from_tensor(self, ref_tensor):
        return None

    def _ranges(self):
        n_pts, n_w, _ = E.stroke_z_layout(self.num_paths, self.stroke_length)
        return n_pts, n_pts + n_w

    def points(self):
        """[num_paths, 3 stroke_length + 1, 2] view of z."""
        return self.z[:self._ranges()[0]].view(self.num_paths, 3 * self.stroke_length + 1, 2)

    def widths(self):
        a, b = self._ranges()
        return self.z[a:b]

    def paper(self):
        return self.z[self._ranges()[1]:]

    def synth(self, cur_iteration):
        """The render of cur_iteration's sample positions composited over white, [1, 3, H, W]."""
        eng = self.session.engine
        eng.set_synth_iteration(cur_iteration)
        self.img = eng.synth(self.z)
        return self.img

    @torch.no_grad()
    def to_image(self):
        """The current geometry rendered with the session's iteration, as linedrawer.py:168-177 converts it (x 254)."""
        from PIL import Image
        img = self.synth(self.session.cur_iteration)
        arr = np.uint8(np.clip(img[0].detach().cpu().numpy().transpose(1, 2, 0), 0, 1) * 254)
        return Image.fromarray(arr, mode="RGB")

    def clip_z(self):
        with torch.no_grad():
            self.widths().clamp_(1.0, self.max_width)  # the stroke colours are fixed black, not part of z

    def get_z(self):
        """The packed parameters.  The reference returns None and optimises its tensors through get_opts; the engine
        needs one vector, as for FftDrawer."""
        return self.z

    def set_z(self, new_z):
        with torch.no_grad():
            return self.z.copy_(new_z.reshape(self.z.shape))

    def get_z_copy(self):
        return None  # as the reference (linedrawer.py:189-190): no best state is ever restored


class VdiffDrawer(DrawingInterface):
    """vdiff.py:58-190 (cc12m_1): z = the noisy image x; synth = one v-prediction step + ClampWithGrad; after every
    optimiser step the loop re-noises x (`makenoise`, pixray.py:1489-1495) and builds a fresh Adam."""

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--vdiff_model", type=str, help="VDIFF model from [yfcc_2, yfcc_1, cc12m_1, cc12m_1_cfg]", default="yfcc_2", dest="vdiff_model")
        parser.add_argument("--vdiff_schedule", type=str, help="VDIFF schedule [default, log]", default="default", dest="vdiff_schedule")
        parser.add_argument("--vdiff_skip", type=float, help="skip a percentage of the way into the decay schedule (0-100)", default=0, dest="vdiff_skip")
        return parser

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        self.iterations = settings.iterations
        self.vdiff_skip = getattr(settings, "vdiff_skip", 0)
        if getattr(settings, "vdiff_schedule", "default") != "default":
            raise NotImplementedError("only the default (spliced DDPM/cosine) schedule is implemented")
        self.clip_model = "ViT-B/16"  # cc12m_1.py:111
        self.x = None

    def load_model(self, settings, device):
        self.device = device

    def get_opts(self, decay_divisor):
        return None

    def get_num_resolutions(self):
        return None

    def init_from_tensor(self, init_tensor, seed=None):
        from .util import vdiff_schedule
        eng = self.session.engine
        self.steps, self.alphas, self.sigmas = vdiff_schedule(self.iterations, self.vdiff_skip)
        eng.vdiff_set_schedule(self.steps, self.alphas, self.sigmas)
        g = None if seed is None else torch.Generator(device=eng.device).manual_seed(seed)
        self.x = torch.randn(eng.z_shape, device=eng.device, generator=g)
        if init_tensor is not None:  # vdiff.py:131-143: x = frame * alpha_0 + noise * sigma_0
            self.x = self.gen_frame(init_tensor) * float(self.alphas[0]) + self.x * float(self.sigmas[0])
        self.x = self.x.contiguous()

    def gen_frame(self, init_tensor):
        """The reverse centre crop (vdiff.py:131-139): a canvas-size start image placed into a zero gen-size frame at the
        margins synth crops away; a gen-size one (no margins) is the frame itself."""
        eng = self.session.engine
        gh, gw = eng.z_shape[2], eng.z_shape[3]
        h, w = eng.image_hw
        t = init_tensor.to(eng.device, torch.float32).reshape(1, 3, h, w)
        if (gh, gw) == (h, w):
            return t
        my, mx = (gh - h) // 2, (gw - w) // 2
        frame = torch.zeros(eng.z_shape, device=eng.device, dtype=torch.float32)
        frame[:, :, my:my + h, mx:mx + w] = t
        return frame

    def set_clip_embed(self, clip_embed):
        """sample_state[3] = {"clip_embed": ...} (pixray.py:880-885)."""
        self.session.engine.vdiff_set_clip_embed(torch.as_tensor(clip_embed).detach().cpu().numpy())

    def makenoise(self, cur_it):
        noise = torch.randn_like(self.x)
        return self.session.engine.vdiff_renoise(self.x, cur_it, noise)

    def synth(self, cur_iteration):
        """The canvas image: the engine crops the clamped prediction to the canvas window (vdiff.py:165-170)."""
        self.session.engine.vdiff_set_iteration(cur_iteration)
        return self.session.engine.synth(self.x)

    def clip_z(self):
        return None

    def get_z(self):
        return self.x

    def set_z(self, new_z):
        with torch.no_grad():
            return self.x.copy_(new_z)

    def get_z_copy(self):
        return self.x.clone()


class SuperResolutionDrawer(DrawingInterface):
    """super_resolution.py:34-107 (with real_esrganer.py at tile 0 / pre_pad 0 / scale 4): z = a quarter-size image in
    [0, 1], synth = clamp_with_grad(RRDBNet(z), 0, 1) on the engine (PXR_DRAWER_SUPERRES), Adam at the global learning
    rate, clip_z clamps z to [0, 1]."""

    models = ("RealESRGAN_x4plus",)  # superresolution_checkpoint_table (super_resolution.py:12-14)

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--super_resolution_model", type=str, help="Super resolution model", default="RealESRGAN_x4plus", dest="super_resolution_model")
        return parser

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        self.super_resolution_model = SuperResolutionDrawer.check_model(settings.super_resolution_model)
        self.z = None

    @staticmethod
    def check_model(name):
        """The reference looks the name up in its checkpoint table: any other name raises (KeyError there)."""
        if name not in SuperResolutionDrawer.models:
            raise ValueError(f"super_resolution_model '{name}' is not in the checkpoint table {list(SuperResolutionDrawer.models)}")
        return name

    def load_model(self, settings, device):
        self.device = device

    def get_opts(self, decay_divisor):
        return None

    def get_num_resolutions(self):
        return None

    def get_z_from_tensor(self, ref_tensor):
        """F.interpolate((t + 1) / 2, size=shape // 4, bilinear, align_corners=False) (super_resolution.py:75-76)."""
        return F.interpolate((ref_tensor + 1) / 2, size=(torch.tensor(ref_tensor.shape[-2:]) // 4).tolist(),
                             mode="bilinear", align_corners=False)

    def init_from_tensor(self, init_tensor):
        """A start image is required: the reference fails on None, here init_tensor None raises ValueError."""
        if init_tensor is None:
            raise ValueError("the super_resolution drawer starts from an image: init_from_tensor needs a tensor")
        z = self.get_z_from_tensor(init_tensor)
        if tuple(z.shape) != tuple(self.session.engine.z_shape):
            raise ValueError(f"the start image gives a latent of shape {tuple(z.shape)}; the engine was built for "
                             f"{tuple(self.session.engine.z_shape)}")
        self.z = z.to(self.session.engine.device, torch.float32).contiguous()

    def reapply_from_tensor(self, new_tensor):
        new_z = self.get_z_from_tensor(new_tensor)
        with torch.no_grad():
            self.z.copy_(new_z)

    def synth(self, cur_iteration):
        return self.session.engine.synth(self.z)

    def clip_z(self):
        with torch.no_grad():
            self.z.copy_(self.z.clip(0, 1))

    def get_z(self):
        return self.z

    def set_z(self, new_z):
        if self.z is None:
            self.z = new_z.detach().to(self.session.engine.device, torch.float32).contiguous().clone()
            return self.z
        with torch.no_grad():
            return self.z.copy_(new_z)

    def get_z_copy(self):
        return self.z.clone()


class FftDrawer(DrawingInterface):
    """fftdrawer.py:13-109, `fft_use="fft"`: params = the rfft2 spectrum [1, 3, H, W/2+1, 2] ~ N(0, 0.01^2)
    (aphantasia fft_image), synth = to_valid_rgb(fft_image)(contrast=0.9); the drawer owns its Adam (lr fft_lrate /
    decay_divisor, fftdrawer.py:63-67), which `get_opts` reports as a learning rate for the engine's fused Adam."""

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--fft_use", type=str, help="use fft or dwt or pixel", default="fft", dest="fft_use")
        parser.add_argument("--fft_decay", default=1.5, type=float, dest="fft_decay")
        parser.add_argument("--fft_wave", default="coif2", help="wavelets: db[1..], coif[1..], haar, dmey", dest="fft_wave")
        parser.add_argument("--fft_sharp", default=0.3, type=float, dest="fft_sharp")
        parser.add_argument("--fft_colors", default=1.5, type=float, dest="fft_colors")
        parser.add_argument("--fft_lrate", default=0.3, type=float, help="Learning rate", dest="fft_lrate")
        return parser

    def __init__(self, settings, session: Session):
        super().__init__(settings)
        self.session = session
        if getattr(settings, "fft_use", "fft") != "fft":
            raise NotImplementedError("fft_use: only 'fft' is on the hot-path scope (dwt / pixel need pytorch_wavelets)")
        self.lrate = getattr(settings, "fft_lrate", 0.3)
        self.params = None

    def load_model(self, settings, device):
        self.device = device

    def get_opts(self, decay_divisor=1):
        return [{"lr": self.lrate / decay_divisor}]

    def get_num_resolutions(self):
        return None

    def init_from_tensor(self, init_tensor, seed=None):
        if init_tensor is not None:
            raise NotImplementedError("resuming the spectrum from an image (fft_image(resume=...)) is init-time and not built")
        eng = self.session.engine
        g = None if seed is None else torch.Generator(device=eng.device).manual_seed(seed)
        self.params = (0.01 * torch.randn(eng.z_shape, device=eng.device, generator=g)).contiguous()  # fft_image(sd=0.01)

    def synth(self, cur_iteration):
        return self.session.engine.synth(self.params)

    def clip_z(self):
        pass

    def get_z(self):
        return self.params  # the reference returns None here and optimises self.params through its own Adam

    def set_z(self, new_z):
        with torch.no_grad():
            return self.params.copy_(new_z)

    def get_z_copy(self):
        return self.params.clone()


class MakeCutouts:
    """pixray.py:399-511.  `transforms` is the per-iteration cache of composed 3x3s (pixray.py:498); when it is None
    a fresh set is sampled (the distributions of the reference's augmentation stacks, pixray_b200/cutouts.py)."""

    def __init__(self, cut_size, cutn, session: Session, cut_pow=1.0, seed=0, aspect=1.0, cut_set=0):
        self.cut_size, self.cutn, self.cut_pow = cut_size, cutn, cut_pow
        self.cut_set = cut_set  # the engine's cutout set of this resolution (set 0: the first perceptor's)
        self.aspect = aspect  # global_aspect_width (pixray.py:402, 1931)
        self.cutn_zoom = int(0.6 * cutn)
        self.noise_fac = 0.1
        self.transforms = None
        self.color_jitter = None
        self.session = session
        self._rng = np.random.default_rng(seed)

    def __call__(self, input, spot=None):
        return self.forward(input, spot)

    def forward(self, input, spot=None):
        if spot is not None:
            raise NotImplementedError("spot prompts are off by default and out of scope (SURVEY.md 8f-2)")
        s = self.session
        if self.transforms is None:
            self.transforms = torch.from_numpy(
                cut_sampler.sample_transforms(self.cutn, self.cut_size, int(self._rng.integers(1 << 31)), aspect=self.aspect))
            # the live stacks end in K.ColorJitter (pixray.py:416, 436); replays of the cached transforms within the
            # same iteration (pixray.py:480-486) do not repeat it
            jitter = cut_sampler.sample_color_jitter(self.cutn, int(self._rng.integers(1 << 31)))
        else:
            jitter = None
        self.color_jitter = jitter
        pad = E.PAD_REFLECTION if s.global_padding_mode == "reflection" else E.PAD_BORDER
        facs = noise = None
        if self.noise_fac:
            facs = (self._rng.random(self.cutn) * self.noise_fac).astype(np.float32)        # pixray.py:509
            noise = torch.randn(self.cutn, 3, self.cut_size, self.cut_size, device=s.engine.device)  # pixray.py:510
        kw = dict(cut_set=self.cut_set) if self.cut_set else {}
        return s.engine.make_cutouts(input, transforms=self.transforms.numpy(), zoom_padding=pad,
                                     fill=s.global_fill_color, noise_facs=facs, noise=noise, it=s.cur_iteration,
                                     color_jitter=jitter, **kw)


class Perceptor:
    """CLIP_Base surface (slip.py:44-74): input_resolution, output_dim, encode_image -> unit-norm [N, D]."""

    def __init__(self, session: Session, clip_idx=0, family="clip", bpe_vocab=None):
        """family: "clip" (openai-CLIP, clip.tokenize) or "slip" (SLIP's SimpleTokenizer), the tokenizer's over-length
        rule; bpe_vocab: path of bpe_simple_vocab_16e6.txt.gz (None: tokenizer.find_vocab looks for it)."""
        self.session, self.clip_idx = session, clip_idx
        self.device = session.engine.device
        c = session.engine.cfg.clip[clip_idx]
        self.input_resolution, self.output_dim = c.image_res, c.out_dim
        self.family, self.bpe_vocab = family, bpe_vocab

    def encode_image(self, imgs, input_range=None, apply_preprocess=True):
        if input_range is not None or not apply_preprocess:
            raise NotImplementedError("only the default preprocess path of the hot loop is implemented (pixray.py:1295)")
        e = self.session.engine.encode_image(self.clip_idx, imgs)
        self.session.last_embeds[self.clip_idx] = e
        return e

    def has_text_tower(self):
        tower = getattr(self.session.engine, "text_tower", None)
        return tower is not None and tower(self.clip_idx) is not None

    def encode_text(self, text):
        """CLIP_Base / SLIP_Base.encode_text (slip.py:68-70, 159-163): str or list of str -> [n, D] float embeddings
        (not normalised), tokenised by this perceptor's family and encoded by the engine's text tower."""
        if not self.has_text_tower():
            raise NotImplementedError("this perceptor has no text tower: load the whole CLIP / SLIP state_dict "
                                      "(token_embedding.weight, positional_embedding, transformer.resblocks.*, ln_final.*, "
                                      "text_projection next to visual.*) before finalize, or pass prompt embeddings")
        tok = tokenizer.get(tokenizer.find_vocab(self.bpe_vocab))
        return self.session.engine.encode_text(self.clip_idx, tok(text, self.family))


class Prompt:
    """pixray.py:268-280.  Instances register themselves with the engine so the loss and its gradient stay on device."""

    def __init__(self, embed, weight=1.0, stop=float("-inf")):
        self.embed = torch.as_tensor(embed, dtype=torch.float32).reshape(-1, torch.as_tensor(embed).shape[-1])
        self.weight = torch.as_tensor(float(weight))
        self.stop = torch.as_tensor(float(stop))
        self._session, self._clip_idx, self._index = None, 0, 0

    @staticmethod
    def register(session: Session, clip_idx, prompts):
        """pmsTable[clip_model] = [Prompt, ...] (pixray.py:859-915)."""
        if any(p.embed.shape[0] != 1 for p in prompts):
            raise ValueError("one embedding row per registered Prompt; image prompts ([cutn, D] rows, refreshed every "
                             "iteration) go through engine.set_image_prompts")
        session.engine.set_prompts(clip_idx, torch.cat([p.embed for p in prompts]).numpy(),
                                   [float(p.weight) for p in prompts], [float(p.stop) for p in prompts])
        for i, p in enumerate(prompts):
            p._session, p._clip_idx, p._index = session, clip_idx, i

    def __call__(self, input):
        return self.forward(input)

    def forward(self, input):
        if self._session is None:
            raise RuntimeError("Prompt.register(session, clip_idx, prompts) must be called first")
        # `input` is normally the tensor perceptor.encode_image just returned (possibly through .float()): the engine still
        # holds those embeddings un-normalised, which its backward needs, so they are not passed back in.  Foreign
        # embeddings are scored as given into scratch buffers: they have no graph behind them, and the engine's own
        # embeddings / gradient (what Session.backward() propagates) are left untouched.
        own = self._session.last_embeds.get(self._clip_idx)
        mine = own is not None and input.data_ptr() == own.data_ptr() and input.shape == own.shape
        return self._session.engine.prompt_loss(self._clip_idx, None if mine else input)[self._index]


def parse_prompt(prompt):
    """pixray.py:290-321: text, text:weight or text:weight:stop."""
    def is_number(s):
        try:
            float(s)
            return True
        except ValueError:
            return False

    text, weight, stop = prompt, 1, float("-inf")
    extra = []
    keep = True
    while len(extra) < 2 and keep:
        vals = text.rsplit(":", 1)
        if len(vals) > 1 and is_number(vals[1]):
            extra.append(float(vals[1]))
            text = vals[0]
        else:
            keep = False
    if len(extra) == 1:
        weight = extra[0]
    elif len(extra) == 2:
        weight, stop = extra[1], extra[0]
    return text, weight, stop


from .util import get_learning_rate_drops  # noqa: E402,F401  (pixray.py:1999-2003)


class Optimizer:
    """optim.<name>([drawer.get_z()], lr) as rebuild_optimisers builds it (pixray.py:520-555): zero_grad / step.  name is
    one of the reference's args.optimiser values the engine runs (E.OPTIMISERS: Adam, AdamW, Adagrad, Adamax,
    DiffGrad), each with its constructor defaults."""

    def __init__(self, session: Session, drawer, lr, name="Adam"):
        if name not in E.OPTIMISERS:
            raise NotImplementedError(f"optimiser {name!r} is not built; available: {sorted(E.OPTIMISERS)}")
        self.session, self.drawer, self.lr = session, drawer, lr
        session.use_optimizer(E.OPTIMISERS[name])

    def zero_grad(self):
        z = self.drawer.get_z()
        z.grad = None

    def step(self):
        z = self.drawer.get_z()
        if getattr(z, "grad", None) is not None:  # the gradient the loop accumulated (several passes when batches > 1)
            self.session.engine.set_z_grad(z.grad.contiguous())
        self.session.engine.step(z, self.lr, self.session.cur_iteration)


def train_iteration(session: Session, drawer, make_cutouts, perceptors, prompt_table, opt):
    """The body of train()/ascend_txt for the default settings (pixray.py:1243-1406, 1436-1512), expressed with the
    plugin objects exactly like the reference does.  make_cutouts: one MakeCutouts, or the cutoutsTable {cut_size:
    MakeCutouts} of perceptors with different input resolutions (pixray.py:1266-1268: every entry cuts the same image,
    each perceptor encodes its own resolution's cutouts).  Returns the list of scalar losses."""
    table = make_cutouts if isinstance(make_cutouts, dict) else None
    have = table.keys() if table else [getattr(make_cutouts, "cut_size", None)]
    for p in perceptors:
        res = getattr(p, "input_resolution", None)
        if None not in have and res is not None and res not in have:
            raise ValueError(f"a perceptor with input resolution {res} needs a MakeCutouts of that size "
                             f"(have {sorted(have)}): pass the cutoutsTable {{cut_size: MakeCutouts}} (pixray.py:642-649)")
    opt.zero_grad()
    out = drawer.synth(session.cur_iteration)
    cur_cutouts = {cs: mc(out) for cs, mc in table.items()} if table else None
    cutouts = None if table else make_cutouts(out)
    result = []
    for i, perceptor in enumerate(perceptors):
        iii = perceptor.encode_image(cur_cutouts[perceptor.input_resolution] if table else cutouts).float()
        for prompt in prompt_table[i]:
            result.append(prompt(iii))
    for mc in (table.values() if table else [make_cutouts]):
        mc.transforms = None  # clear the per-iteration cache (pixray.py:1339-1342)
    session.backward(drawer)
    opt.step()
    drawer.clip_z()
    if isinstance(drawer, VdiffDrawer) and session.cur_iteration >= 1:
        # pixray.py:1489-1495: re-noise x for the next timestep and start a fresh Adam (whatever args.optimiser chose)
        # with the schedule's step size
        it = session.cur_iteration
        lr = float(drawer.sigmas[it] / drawer.alphas[it])
        drawer.makenoise(it)
        opt.lr = min(lr * 0.001, 0.01)
        session.use_optimizer(E.OPT_ADAM)
    return result
