"""Host-side geometry of the pixel drawer's shaped cells (PixelDrawer, pixeldrawer.py:110-304): the grid size, the cell
polygons in draw order and the initial fill colours sampled from a start image.

The engine renders these polygons (PXR_DRAWER_POLYGON) and optimises only their colours, so everything here runs once at
init.  The arithmetic follows the reference's order of operations -- Python floats for the cell corners and the
interpolated vertex positions, rounded to float32 at the end, float32 sums for the colours -- so the vertices match
the reference bit for bit (tests/golden/pixel_shapes.npz).

One deliberate difference: the reference draws squares for a `pixel_type` it does not know; here that is refused.
"""
import numpy as np

PIXEL_TYPES = ("rect", "rectshift", "hex", "tri", "diamond", "knit")
SHIFT_TYPES = ("hex", "rectshift", "diamond")  # every other row has one cell less, offset by half a cell
MAX_VERTICES = 8  # knit
MAX_COLOUR_SUBSAMPLES = 4  # per axis and cell (encode_image)


def check_pixel_type(pixel_type):
    if pixel_type not in PIXEL_TYPES:
        raise ValueError(f"pixel_type '{pixel_type}' is not one of {', '.join(PIXEL_TYPES)}")
    return pixel_type


def grid_for(size, pixel_type="rect", pixel_size=None, pixel_scale=None, edge_check=True, iso_check=True, verbose=True):
    """(num_rows, num_cols) as PixelDrawer.__init__ derives them (pixeldrawer.py:123-177).  size = (width, height);
    pixel_size = (cols, rows) overrides the 40x40 / 40x50 / 80x45 defaults.  With iso_check and no pixel_size, tri cells
    get 1.414x the columns, hex cells 1.414x the rows and diamonds twice the rows.  Then pixel_scale divides, the counts
    are clamped to the canvas, and edge_check makes the counts odd (shift types) or odd columns and even rows (tri)."""
    check_pixel_type(pixel_type)
    canvas_width, canvas_height = size
    if pixel_size is not None:
        num_cols, num_rows = pixel_size
    elif canvas_width == canvas_height:
        num_cols, num_rows = 40, 40
    elif canvas_width < canvas_height:
        num_cols, num_rows = 40, 50
    else:
        num_cols, num_rows = 80, 45
    if iso_check and pixel_size is None:
        if pixel_type == "tri":
            num_cols = int(1.414 * num_cols)
        elif pixel_type == "hex":
            num_rows = int(1.414 * num_rows)
        elif pixel_type == "diamond":
            num_rows = int(2 * num_rows)
    if pixel_scale is not None and pixel_scale > 0:
        num_cols, num_rows = int(num_cols / pixel_scale), int(num_rows / pixel_scale)
    shrink = False
    if num_cols > canvas_width:
        shrink, num_cols = True, canvas_width
    if num_rows > canvas_height:
        shrink, num_rows = True, canvas_height
    if verbose:
        if shrink:
            print("pixel grid size should not be larger than output pixel size: reducing pixel grid")
        print(f"Running pixeldrawer with {num_cols}x{num_rows} grid")  # before the edge check, like the reference
    if edge_check:
        if pixel_type in SHIFT_TYPES:
            num_cols += 1 - num_cols % 2
            num_rows += 1 - num_rows % 2
        elif pixel_type == "tri":
            num_cols += 1 - num_cols % 2
            num_rows += num_rows % 2
    return num_rows, num_cols


def _cells(num_rows, num_cols, pixel_type):
    """(row, column, column offset) of every cell in draw order."""
    for r in range(num_rows):
        if pixel_type in SHIFT_TYPES and r % 2 == 0:
            n, off = num_cols - 1, 0.5
        else:
            n, off = num_cols, 0
        for c in range(n):
            yield r, c, off


def _lerp(t, a, b):
    """a + t (b - a) in the reference's operation order: t * (b - a) + a (map_number, pixeldrawer.py:28-29)."""
    return t * (b - a) + a


def _vertices(pixel_type, x1, y1, x2, y2, r, c):
    """The polygon of one cell with corners (x1, y1), (x2, y2) (the *_from_corners helpers, pixeldrawer.py:21-94)."""
    if pixel_type == "hex":  # pointy-top hexagon reaching 1/6 of the cell height above and below it
        ya, yb, yc, yd = (_lerp(t, y1, y2) for t in (7 / 6, 5 / 6, 1 / 6, -1 / 6))
        xh = _lerp(0.5, x1, x2)
        return [(xh, ya), (x1, yb), (x1, yc), (xh, yd), (x2, yc), (x2, yb)]
    if pixel_type == "diamond":  # twice the cell height, centred on it
        ya, yb, yh = _lerp(-0.5, y1, y2), _lerp(1.5, y1, y2), _lerp(0.5, y1, y2)
        xh = _lerp(0.5, x1, x2)
        return [(xh, ya), (x1, yh), (xh, yb), (x2, yh)]
    if pixel_type == "tri":  # twice the cell width; up and down alternate like a checkerboard
        xa, xb, xh = _lerp(1.5, x1, x2), _lerp(-0.5, x1, x2), _lerp(0.5, x1, x2)
        if (r + c) % 2 == 0:
            return [(xh, y1), (xb, y2), (xa, y2)]
        return [(xh, y2), (xa, y1), (xb, y1)]
    if pixel_type == "knit":  # a V-shaped stitch leaning up into the row above
        xm = (x1 + x2) / 2.0
        up1, up2 = _lerp(0.45, y2, y1), _lerp(1 + 0.45, y2, y1)
        down1, down2 = _lerp(0.30, y1, y2), _lerp(1 + 0.30, y1, y2)
        back1, back2 = _lerp(0.2, x2, xm), _lerp(0.2, x1, xm)
        return [(xm, down2), (x2, up1), (x2, up2), (back1, up2), (xm, down1), (back2, up2), (x1, up2), (x1, up1)]
    return [(x1, y1), (x2, y1), (x2, y2), (x1, y2)]  # rect, rectshift


def polygons(size, num_rows, num_cols, pixel_type):
    """Cell polygons in draw order (later ones are drawn over earlier ones): xy float32 [total_vertices, 2] in canvas
    pixels and offsets int32 [n + 1], polygon k = xy[offsets[k]:offsets[k + 1]]."""
    check_pixel_type(pixel_type)
    canvas_width, canvas_height = size
    cell_width, cell_height = canvas_width / num_cols, canvas_height / num_rows
    pts, offsets = [], [0]
    for r, c, off in _cells(num_rows, num_cols, pixel_type):
        x, y = (off + c) * cell_width, r * cell_height
        v = _vertices(pixel_type, x, y, x + cell_width, y + cell_height, r, c)
        pts.extend(v)
        offsets.append(len(pts))
    return np.asarray(pts, dtype=np.float32).reshape(-1, 2), np.asarray(offsets, dtype=np.int32)


def init_colours(init_tensor, num_rows, num_cols, pixel_type):
    """Initial RGBA fills (encode_image, pixeldrawer.py:200-271): each cell averages up to 4 x 4 pixels of
    (init_tensor + 1) / 2 ([1, 3, h, w] in [-1, 1]) on a subsample lattice starting at the cell's top-left corner, with
    the reference's int() truncations; alpha 1.  float32 [n, 4]."""
    check_pixel_type(pixel_type)
    if init_tensor is None:
        raise ValueError("the pixel drawer's shaped cells take their colours from a start image: pass an init_image or "
                         "use init_noise (the reference has no random start for them either)")
    t = init_tensor.detach().cpu().numpy() if hasattr(init_tensor, "detach") else np.asarray(init_tensor)
    img = (t[0].astype(np.float32) + np.float32(1.0)) / np.float32(2.0)
    h, w = img.shape[1], img.shape[2]
    cw, ch = w / num_cols, h / num_rows

    def lattice(cell):
        if int(cell) < MAX_COLOUR_SUBSAMPLES:
            return list(range(int(cell)))
        step = cell / MAX_COLOUR_SUBSAMPLES
        return [int(i * step) for i in range(MAX_COLOUR_SUBSAMPLES)]

    sub_x, sub_y = lattice(cw), lattice(ch)
    cells = list(_cells(num_rows, num_cols, pixel_type))
    n = len(cells)
    acc = np.zeros((n, 3), dtype=np.float32)
    count = np.zeros(n, dtype=np.int64)
    base_x = np.array([(off + c) * cw for (_, c, off) in cells], dtype=np.float64)
    base_y = np.array([int(r * ch) for (r, _, _) in cells], dtype=np.int64)
    for tx in sub_x:  # the reference's loop order (x outer, y inner): float32 sums in the same sequence
        sx = base_x + tx
        for ty in sub_y:
            sy = base_y + ty
            ok = (sx < w) & (sy < h)
            vals = img[:, np.where(ok, sy, 0), np.where(ok, sx, 0).astype(np.int64)].T
            acc += np.where(ok[:, None], vals, np.float32(0.0))
            count += ok
    count = np.maximum(count, 1)  # an empty cell keeps colour 0, as in the reference
    out = np.ones((n, 4), dtype=np.float32)
    out[:, :3] = acc / count[:, None].astype(np.float32)
    return out
