"""pixray's filter plugins (filters/FilterInterface.py:4-16 and filters/{tiler,wallpaper,colorlookup}.py) on the H100 engine.

The reference applies them to drawer.synth's output before MakeCutouts (do_synth_and_filter, pixray.py:1203-1222): each is an
nn.Module whose forward(img) returns (img, loss).  Here a filter instance describes itself to the engine (pxr_add_filter): the
image transform, its adjoint and the loss gradient run inside pxr_iterate; `forward` is not called in the fused loop."""
from . import engine as E

default_color_table = [[0, 0, 0], [255, 255, 255], [63, 40, 50], [38, 43, 68], [90, 105, 136], [139, 155, 180], [25, 60, 62],
                       [38, 92, 66], [62, 137, 72], [99, 199, 77], [254, 231, 97], [254, 174, 52], [254, 174, 52], [247, 118, 34],
                       [184, 111, 80], [116, 63, 57]]  # colorlookup.py:10-26 (0..255)


class FilterInterface:
    """filters/FilterInterface.py."""
    kind = None

    @staticmethod
    def add_settings(parser):
        return parser

    def __init__(self, settings, device=None):
        self.device = device
        self._session = None
        self._index = None

    def engine_params(self, settings):
        return []

    def attach(self, session, settings, weight=1.0):
        """filterClasses.append({"filter": filtInstance, "weight": weight}) (pixray.py:664) for the engine."""
        self._session = session
        self._index = session.engine.add_filter(self.kind, weight, self.engine_params(settings))
        return self

    def forward(self, img):
        raise NotImplementedError("filters run inside the engine's fused iteration (pxr_add_filter); there is no per-call path")


class TilerFilter(FilterInterface):
    """filters/tiler.py: random tiled shifts in x and y, no loss."""
    kind = E.FILTER_TILER


class WallpaperFilter(FilterInterface):
    """filters/wallpaper.py."""
    kind = E.FILTER_WALLPAPER
    _types = {None: 0, "none": 0, "shift": 1, "horizontal": 2, "vertical": 3}

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--wallpaper_type", type=str, help="none, shift, horizontal", default=None, dest="wallpaper_type")
        parser.add_argument("--wallpaper_edge_match", type=int, help="force repeating match in pixels", default=0, dest="wallpaper_edge_match")
        return parser

    def __init__(self, settings, device=None):
        super().__init__(settings, device)
        self.wallpaper_type = settings.wallpaper_type
        self.edge_match = settings.wallpaper_edge_match

    def engine_params(self, settings):
        # any other string falls into the reference's final `else` branch (wallpaper.py:69): both directions
        return [self._types.get(self.wallpaper_type, 0), self.edge_match]


class ColorLookup(FilterInterface):
    """filters/colorlookup.py: maps to a fixed colour table (args.palette, else the built-in 16 colours)."""
    kind = E.FILTER_LOOKUP

    @staticmethod
    def add_settings(parser):
        parser.add_argument("--lookup_beta", type=float, help="loss scaling", default=10.0, dest="lookup_beta")
        return parser

    def __init__(self, settings, device=None):
        super().__init__(settings, device)
        self.beta = settings.lookup_beta
        table = settings.palette
        if table is None:
            print("WARNING: using built in palette")
            table = [[c / 255.0 for c in rgb] for rgb in default_color_table]
        self.color_table = [list(map(float, rgb)) for rgb in table]

    def engine_params(self, settings):
        return [self.beta] + [v for rgb in self.color_table for v in rgb]


filters_class_table = {"lookup": ColorLookup, "tiler": TilerFilter, "wallpaper": WallpaperFilter}  # pixray.py:55-59
