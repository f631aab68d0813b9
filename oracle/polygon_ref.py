"""float64 restatement of diffvg's render of PixelDrawer's scene (pixeldrawer.py:339-342) for the tests: closed polygons
filled with the even-odd rule, every fill opaque, the topmost polygon containing a sample wins, an uncovered sample is
transparent black, and a pixel is the mean of its samples (the box filter of radius 0.5 weighs them equally).

Sample positions are explicit ([H, W, S, 2] canvas coordinates, sample s of pixel (x, y) inside [x, x + 1] x
[y, y + 1]): the engine's own (pxr_test_raster_samples) for the parity tests, a regular lattice for the area checks.
Pure numpy / torch; no GPU and no reference checkout needed.
"""
import numpy as np
import torch


def _even_odd(v, px, py):
    """Even-odd containment of the points (px, py) in polygon v [m, 2], by the same crossing test as the kernel
    (kernels_raster.cu): the sign of a cross product, exact in float64 for float32 inputs."""
    inside = np.zeros(px.shape, dtype=bool)
    m = len(v)
    for i in range(m):
        xi, yi = v[i]
        xj, yj = v[i - 1]
        cross = (xj - xi) * (py - yi) - (px - xi) * (yj - yi)
        hit = ((yi > py) != (yj > py)) & ((cross > 0) if yj > yi else (cross < 0))
        inside ^= hit
    return inside


def _edge_distance(v, px, py):
    d = np.full(px.shape, np.inf)
    m = len(v)
    for i in range(m):
        ax, ay = v[i - 1]
        bx, by = v[i]
        ex, ey = bx - ax, by - ay
        ll = ex * ex + ey * ey
        t = np.clip(((px - ax) * ex + (py - ay) * ey) / ll, 0.0, 1.0) if ll > 0 else np.zeros(px.shape)
        d = np.minimum(d, np.hypot(px - (ax + t * ex), py - (ay + t * ey)))
    return d


def polygon_winners(verts, offsets, H, W, samples, edge_distance=False):
    """winner [S, H, W] int64: index of the topmost polygon containing each sample, -1 where none does.  With
    edge_distance, also [S, H, W] float64: the distance of each sample to the nearest edge of any polygon (inf when no
    edge lies within a pixel of it) -- samples that close to an edge may legitimately go either way."""
    verts = np.asarray(verts, dtype=np.float64)
    offsets = np.asarray(offsets)
    s = np.asarray(samples, dtype=np.float64)
    S = s.shape[2]
    win = np.full((H, W, S), -1, dtype=np.int64)
    dist = np.full((H, W, S), np.inf) if edge_distance else None
    for k in range(len(offsets) - 1):  # draw order: a later polygon overwrites an earlier one
        v = verts[offsets[k]:offsets[k + 1]]
        x0, y0 = v.min(axis=0)
        x1, y1 = v.max(axis=0)
        # samples of pixel x lie in [x, x + 1]: the pixels that can hold samples inside the box, one more each side
        # for the edge distance
        px0, px1 = max(0, int(np.floor(x0)) - 2), min(W - 1, int(np.floor(x1)) + 1)
        py0, py1 = max(0, int(np.floor(y0)) - 2), min(H - 1, int(np.floor(y1)) + 1)
        if px1 < px0 or py1 < py0:
            continue
        blk = s[py0:py1 + 1, px0:px1 + 1]
        X, Y = blk[..., 0], blk[..., 1]
        inside = _even_odd(v, X, Y)
        w = win[py0:py1 + 1, px0:px1 + 1]
        w[inside] = k
        if edge_distance:
            dd = dist[py0:py1 + 1, px0:px1 + 1]
            np.minimum(dd, _edge_distance(v, X, Y), out=dd)
    win = np.ascontiguousarray(win.transpose(2, 0, 1))
    if edge_distance:
        return win, np.ascontiguousarray(dist.transpose(2, 0, 1))
    return win


def polygon_render(verts, offsets, colours, H, W, samples, winners=None):
    """[3, H, W] float64 torch tensor: the mean over each pixel's samples of the winning polygon's RGB (0 where no polygon
    covers the sample).  Linear in `colours` ([n, 4] RGBA, any float torch tensor): differentiable through autograd.
    `winners` ([S, H, W], from polygon_winners) skips the geometry when the caller already has it."""
    if winners is None:
        winners = polygon_winners(verts, offsets, H, W, samples)
    c = torch.as_tensor(colours).to(torch.float64)
    rgb = torch.cat([c[:, :3], torch.zeros(1, 3, dtype=torch.float64, device=c.device)])  # row n: uncovered
    idx = torch.as_tensor(np.where(winners < 0, c.shape[0], winners), device=c.device)
    return rgb[idx].mean(dim=0).permute(2, 0, 1)


def regular_samples(H, W, n):
    """An n x n lattice of sample positions per pixel (cell centres), [H, W, n * n, 2]."""
    o = (np.arange(n) + 0.5) / n
    oy, ox = np.meshgrid(o, o, indexing="ij")
    s = np.empty((H, W, n * n, 2))
    s[..., 0] = np.arange(W)[None, :, None] + ox.reshape(-1)[None, None, :]
    s[..., 1] = np.arange(H)[:, None, None] + oy.reshape(-1)[None, None, :]
    return s
