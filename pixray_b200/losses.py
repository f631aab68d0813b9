"""The reference's auxiliary losses (Losses/*.py, registered in pixray.loss_class_table, pixray.py:131-140) on the H100
engine.  Same class names, `add_settings` arguments and `parse_settings` behaviour as the reference; the difference is
where the arithmetic runs: the reference's `get_loss` returns an autograd tensor, here `attach()` installs the loss
inside the engine (one fused loss + gradient kernel per loss, pixray_b200/csrc/kernels_losses.cu) and `get_loss`
returns the value the engine computed for the current iteration -- gradients never pass through torch.

    loss = SmoothnessLoss(device=dev); args = loss.parse_settings(args); loss.attach(session, args, weight)
"""
import argparse

import numpy as np
import torch

from . import engine as E


class LossInterface:
    """Losses/LossInterface.py:4-35."""

    def __init__(self, device=None):
        self.device = device
        self._session, self._index = None, None

    def instance_settings(self, arglist):
        pass

    @staticmethod
    def add_settings(parser):
        return parser

    def help(self):
        """One block of text per option this loss registers (LossInterface.py:17-23 returns only the last option's block: it
        assigns inside the loop; the text of every block is kept so that block is still what a caller matching on it finds
        last)."""
        probe = self.add_settings(argparse.ArgumentParser(add_help=False))
        blocks = []
        for action in probe._actions:
            blocks.append("parmeter name: %s\nHelp: %s\nUse case: pixray.add_argument(%s=%s)"
                          % (action.dest, action.help, action.dest, action.default))
        return blocks[-1] if blocks else ""

    def parse_settings(self, args):
        return args

    def add_globals(self, args):
        return {}

    # -- engine side
    kind = None

    def engine_params(self, args, session):
        raise NotImplementedError

    def attach(self, session, args, weight=1.0):
        """lossClasses.append({"loss": lossInstance, "weight": weight}) (pixray.py:979-981) for the engine."""
        self._session = session
        self._index = session.engine.add_aux_loss(self.kind, weight, self.engine_params(args, session))
        return self

    def get_loss(self, cur_cutouts, out, args, globals=None, lossGlobals=None):
        if self._session is None:
            raise RuntimeError(f"{type(self).__name__}.attach(session, args, weight) must be called first")
        return torch.as_tensor(self._session.engine.read_losses()[self._index])


class SymmetryLoss(LossInterface):
    """Losses/SymmetryLoss.py."""
    kind = E.LOSS_SYMMETRY

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--symmetry_weight", type=float, help="how much symmetry is weighted in loss", default=1, dest="symmetry_weight")
        return parser

    def engine_params(self, args, session):
        return [args.symmetry_weight]


class SaturationLoss(LossInterface):
    """Losses/SaturationLoss.py."""
    kind = E.LOSS_SATURATION

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--saturation_weight", type=float, help="strength of pallete loss effect", default=1, dest="saturation_weight")
        return parser

    def engine_params(self, args, session):
        return [args.saturation_weight]


class PaletteLoss(LossInterface):
    """Losses/PaletteLoss.py (args.palette: list of [r, g, b] in [0, 1], pixray.py's palette_from_string output)."""
    kind = E.LOSS_PALETTE

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--palette_weight", type=float, help="strength of pallete loss effect", default=1, dest="palette_weight")
        return parser

    def engine_params(self, args, session):
        pal = np.asarray(args.palette, dtype=np.float32).reshape(-1, 3)
        if pal.shape[0] < 1:
            raise ValueError("palette loss needs at least one colour")
        return [args.palette_weight] + pal.reshape(-1).tolist()


class SmoothnessLoss(LossInterface):
    """Losses/SmoothnessLoss.py."""
    kind = E.LOSS_SMOOTHNESS
    _types = {"default": 0, "clipped": 1, "log": 2}

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--smoothness_weight", type=float, help="strength of smoothness loss effect", default=1, dest="smoothness_weight")
        parser.add_argument("--smoothness_type", type=str, help="enforce smoothness type: default/clipped/log", default="default", dest="smoothness_type")
        parser.add_argument("--smoothness_gaussian_kernel", type=float, help="enforce smoothness aux gaussian blur kernel", default=0, dest="smoothness_gaussian_kernel")
        parser.add_argument("--smoothness_gaussian_std", type=float, help="enforce smoothness aux gaussian blur std", default=1, dest="smoothness_gaussian_std")
        parser.add_argument("--smoothness_spacing", type=int, help="enforce smoothness spacing", default=1, dest="smoothness_spacing")
        parser.add_argument("--smoothness_edge_order", type=int, help="enforce smoothness edge order", default=1, dest="smoothness_edge_order")
        return parser

    def engine_params(self, args, session):
        if getattr(args, "smoothness_gaussian_kernel", 0):
            raise NotImplementedError("smoothness_gaussian_kernel != 0 (pre-blur) is not implemented in the engine")
        if getattr(args, "smoothness_edge_order", 1) != 1:
            raise NotImplementedError("only smoothness_edge_order = 1 is implemented in the engine")
        # any other string falls through to the un-clipped branch in the reference (SmoothnessLoss.py:101-104)
        return [args.smoothness_weight, self._types.get(args.smoothness_type, 0), getattr(args, "smoothness_spacing", 1)]


class EdgeLoss(LossInterface):
    """Losses/EdgeLoss.py with a colour target (edge_input_image / edge_mask_image are file-based variants, not built)."""
    kind = E.LOSS_EDGE

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--edge_thickness", type=int, help="thickness of the edge area all the way around (percent)", default=5, dest="edge_thickness")
        parser.add_argument("--edge_margins", nargs=4, type=int, help="this is for the thickness of each edge (left, right, up, down) 0-pixel size", default=None, dest="edge_margins")
        parser.add_argument("--edge_color", type=str, help="this is the color of the specified region", default="white", dest="edge_color")
        parser.add_argument("--edge_color_weight", type=float, help="how much edge color is enforced", default=0.1, dest="edge_color_weight")
        parser.add_argument("--global_color_weight", type=float, help="how much global color is enforced ", default=0.05, dest="global_color_weight")
        parser.add_argument("--edge_input_image", type=str, help="TBD", default="", dest="edge_input_image")
        parser.add_argument("--edge_mask_image", type=str, help="TBD", default="", dest="edge_mask_image")
        return parser

    def parse_settings(self, args):
        if isinstance(args.edge_color, str):
            c = args.edge_color.strip()
            if c and c[0] in "([":  # util.parse_triple_to_rgb: "(255+255+0)" or "[1+1+0]"
                vals = [float(v) for v in c.strip("()[]").split("+")]
                args.edge_color = [v / 255.0 for v in vals] if c[0] == "(" else vals
            elif c == "white":
                args.edge_color = [1.0, 1.0, 1.0]
            elif c == "black":
                args.edge_color = [0.0, 0.0, 0.0]
            else:
                raise ValueError(f"edge_color '{c}': give an explicit (r+g+b) / [r+g+b] triple (named colours need matplotlib)")
        if args.edge_margins is None:
            t = args.edge_thickness
            args.edge_margins = (t, t, t, t)
        if getattr(args, "edge_input_image", "") or getattr(args, "edge_mask_image", ""):
            raise NotImplementedError("edge_input_image / edge_mask_image are not implemented in the engine")
        return args

    def engine_params(self, args, session):
        H, W = session.engine.image_hw
        left, right, upper, lower = args.edge_margins
        # util.map_number(n, 0, 100, 0, size) then int() (EdgeLoss.py:85-88)
        px = [int(left / 100.0 * W), int(right / 100.0 * W), int(upper / 100.0 * H), int(lower / 100.0 * H)]
        return [args.edge_color_weight, args.global_color_weight] + px + list(args.edge_color)


class GaussianLoss(LossInterface):
    """Losses/GaussianLoss.py."""
    kind = E.LOSS_GAUSSIAN

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--gaussian_weight", type=float, help="gaussian's weight", default=1, dest="gaussian_weight")
        parser.add_argument("--gaussian_std", nargs=2, type=float, help="gaussian's std for both x and y", default=(40, 40), dest="gaussian_std")
        parser.add_argument("--gaussian_color", nargs=3, type=float, help="color for gaussian to optimize to", default=(255, 255, 255), dest="gaussian_color")
        return parser

    def engine_params(self, args, session):
        return [args.gaussian_weight, args.gaussian_std[0], args.gaussian_std[1]] + list(args.gaussian_color)


class AestheticLoss(LossInterface):
    """Losses/AestheticLoss.py.  The reference downloads the linear AVA head to models/ava_vit_b_16_linear.pth
    (AestheticLoss.py:15-20); there is no network here, so the head comes in through the extra setting `aesthetic_head`:
    the path of that .pth file, or the dict it holds ({"weight": [1, D], "bias": [1]}); default = the reference's path."""
    kind = E.LOSS_AESTHETIC
    default_path = "models/ava_vit_b_16_linear.pth"

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--aesthetic_target", type=float, help="0-10", default=10, dest="aesthetic_target")
        parser.add_argument("--aesthetic_head", help="path of ava_vit_b_16_linear.pth, or its {'weight','bias'} dict",
                            default=None, dest="aesthetic_head")
        return parser

    def parse_settings(self, args):
        head = getattr(args, "aesthetic_head", None)
        if head is None:
            head = self.default_path
        if isinstance(head, (str, bytes)) or hasattr(head, "__fspath__"):
            import os
            if not os.path.exists(head):
                raise FileNotFoundError(f"aesthetic loss: linear head '{head}' not found (the reference downloads it from "
                                        "https://dazhi.art/f/ava_vit_b_16_linear.pth; pass aesthetic_head=<path or dict>)")
            head = torch.load(head, map_location="cpu", weights_only=False)  # layer_weights, AestheticLoss.py:23
        if not (isinstance(head, dict) and "weight" in head and "bias" in head):
            raise ValueError("aesthetic_head must hold 'weight' [1, D] and 'bias' [1]")
        args.aesthetic_head = head
        return args

    def engine_params(self, args, session):
        head = args.aesthetic_head
        w = torch.as_tensor(head["weight"], dtype=torch.float32).reshape(-1)
        b = float(torch.as_tensor(head["bias"]).reshape(-1)[0])
        return [args.aesthetic_target, b] + w.tolist()


# pixray.loss_class_table (pixray.py:131-140) restricted to the losses on the hot-path scope (SURVEY.md 8 row a15),
# plus "gaussian" which the reference only reaches through add_custom_loss
loss_class_table = {
    "palette": PaletteLoss, "saturation": SaturationLoss, "symmetry": SymmetryLoss, "smoothness": SmoothnessLoss,
    "edge": EdgeLoss, "aesthetic": AestheticLoss, "gaussian": GaussianLoss,
}
