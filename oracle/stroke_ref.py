"""float64 restatement of the line-sketch render (LineDrawer.synth, linedrawer.py:156-166) and of its boundary gradient,
for the tests.  diffvg is not vendored, so these are the conventions the engine states (DESIGN.md §3) and this module
restates; it does not pin diffvg itself:

- Each cubic segment is flattened into S chords at t = i / S (Bernstein weights).  A path covers the points within its
  stroke width w of one of its chords: the union of round-capped capsules {x : dist(x, chord) <= w}.  w is the half
  width (diffvg's save_svg writes 2 w), so caps and joins are round.
- The paper rectangle is opaque and covers the canvas; every stroke is opaque black, later paths over earlier ones.  A
  sample's RGBA is black (0, 0, 0, 1) when covered, else the paper's RGBA; a pixel is the mean of its samples (box filter
  of radius 0.5), composited as synth does: out = rgb a + (1 - a).
- The backward is the exact derivative of the box-filtered image: with c(p) the covered fraction of pixel p,
  d out / d theta = sum_p G(p) dc(p) / d theta, G(p) = sum_ch g_ch(p) d out_ch / dc at the forward's coverage, and
  dc / d theta = the integral over the visible outline (points of a capsule boundary that no other capsule strictly
  covers) of v_n ds.  On a straight side v_n = ((1 - s) da + s db) . n + dw; on the circle around a vertex v_n = dv . u + dw.
  Sides are walked across the pixel grid and integrate exactly; the vertex circles use ARC_NODES midpoint nodes.  At a
  joint between consecutive chords of a path the circle is counted once (the directions outside both chords' bodies).
  The paper colour gets the interior term d out / d paper at the forward's coverage.

Sample positions are explicit ([H, W, n, 2] canvas coordinates): the engine's own (pxr_test_raster_samples) for the
parity tests, a regular lattice (polygon_ref.regular_samples) for the area and finite-difference checks.
Pure numpy / torch; no GPU needed."""
import math

import numpy as np
import torch

S = 16          # chords per cubic segment
ARC_NODES = 64  # midpoint nodes on a full vertex circle


def bernstein(t):
    t = np.asarray(t, dtype=np.float64)
    u = 1.0 - t
    return np.stack([u * u * u, 3 * t * u * u, 3 * t * t * u, t * t * t])


def flatten(points):
    """points [N, 3L + 1, 2] -> chords [N L S, 4] (ax, ay, bx, by), path-major, then segment, then chord."""
    p = np.asarray(points, dtype=np.float64)
    N, M, _ = p.shape
    L = (M - 1) // 3
    B = bernstein(np.arange(S + 1) / S)  # [4, S + 1]
    out = np.empty((N, L, S, 4))
    for k in range(N):
        for j in range(L):
            V = B.T @ p[k, 3 * j:3 * j + 4]  # [S + 1, 2]
            out[k, j, :, :2] = V[:-1]
            out[k, j, :, 2:] = V[1:]
    return out.reshape(-1, 4)


def cubic_flattening_error(points, n_eval=64):
    """(max distance of the true curve from the flattened polyline, the sagitta bound max|B''| / (8 S^2)) over every
    segment: the chord of [t_i, t_i+1] stays within max|B''| (1 / S)^2 / 8 of the arc it replaces."""
    p = np.asarray(points, dtype=np.float64)
    N, M, _ = p.shape
    err = bound = 0.0
    for k in range(N):
        for j in range((M - 1) // 3):
            P = p[k, 3 * j:3 * j + 4]
            second = np.array([P[0] - 2 * P[1] + P[2], P[1] - 2 * P[2] + P[3]])  # B'' = 6 ((1 - t) d0 + t d1)
            bound = max(bound, 6 * max(np.hypot(*second[0]), np.hypot(*second[1])) / (8 * S * S))
            for i in range(S):
                t = i / S + np.arange(1, n_eval) / (n_eval * S)
                X = bernstein(t).T @ P
                a = bernstein(i / S) @ P
                b = bernstein((i + 1) / S) @ P
                err = max(err, float(np.max(_seg_dist(X[:, 0], X[:, 1], np.concatenate([a, b])))))
    return err, bound


def _seg_dist(px, py, c):
    ex, ey = c[2] - c[0], c[3] - c[1]
    dx, dy = px - c[0], py - c[1]
    ll = ex * ex + ey * ey
    t = np.clip((dx * ex + dy * ey) / ll, 0.0, 1.0) if ll > 0 else np.zeros_like(px)
    return np.hypot(dx - t * ex, dy - t * ey)


def unpack(z, n_paths, n_segments):
    z = np.asarray(z, dtype=np.float64).reshape(-1)
    n_pts = n_paths * (3 * n_segments + 1) * 2
    return z[:n_pts].reshape(n_paths, 3 * n_segments + 1, 2), z[n_pts:n_pts + n_paths], z[n_pts + n_paths:n_pts + n_paths + 4]


def winners(caps, cap_w, cap_path, H, W, samples, edge_distance=False):
    """[n, H, W] int64: the topmost path covering each sample (-1: paper).  With edge_distance, also the distance of each
    sample to the nearest capsule outline ([n, H, W]; inf farther than a pixel): such samples may go either way."""
    s = np.asarray(samples, dtype=np.float64)
    n = s.shape[2]
    win = np.full((H, W, n), -1, dtype=np.int64)
    dist = np.full((H, W, n), np.inf) if edge_distance else None
    for c in range(len(caps)):  # ascending: a later path overwrites an earlier one
        a = caps[c]
        w = cap_w[c]
        x0, x1 = min(a[0], a[2]) - w, max(a[0], a[2]) + w
        y0, y1 = min(a[1], a[3]) - w, max(a[1], a[3]) + w
        px0, px1 = max(0, int(np.floor(x0)) - 2), min(W - 1, int(np.floor(x1)) + 1)
        py0, py1 = max(0, int(np.floor(y0)) - 2), min(H - 1, int(np.floor(y1)) + 1)
        if px1 < px0 or py1 < py0:
            continue
        blk = s[py0:py1 + 1, px0:px1 + 1]
        d = _seg_dist(blk[..., 0], blk[..., 1], a)
        win[py0:py1 + 1, px0:px1 + 1][d <= w] = cap_path[c]
        if edge_distance:
            dd = dist[py0:py1 + 1, px0:px1 + 1]
            np.minimum(dd, np.abs(d - w), out=dd)
    win = np.ascontiguousarray(win.transpose(2, 0, 1))
    if edge_distance:
        return win, np.ascontiguousarray(dist.transpose(2, 0, 1))
    return win


class Scene:
    """The flattened geometry of z (packed [points | widths | paper]) for n_paths x n_segments; `caps` ([N L S, 4], e.g.
    the engine's own fp32 chords) replaces the float64 flattening."""

    def __init__(self, z, n_paths, n_segments, H, W, caps=None):
        self.points, self.widths, self.paper = unpack(z, n_paths, n_segments)
        self.N, self.L, self.H, self.W = n_paths, n_segments, H, W
        self.caps = flatten(self.points) if caps is None else np.asarray(caps, dtype=np.float64).reshape(-1, 4)
        per = n_segments * S
        self.cap_path = np.repeat(np.arange(n_paths), per)
        self.cap_w = self.widths[self.cap_path]
        self.first = np.arange(len(self.caps)) % per == 0
        self.last = (np.arange(len(self.caps)) + 1) % per == 0

    def winners(self, samples, edge_distance=False):
        return winners(self.caps, self.cap_w, self.cap_path, self.H, self.W, samples, edge_distance)


def coverage(win):
    return (np.asarray(win) >= 0).mean(axis=0)


def synth_composite(rgba):
    """LineDrawer.synth on a rendered [H, W, 4] RGBA image: rgb a + 1 (1 - a), NHWC -> [1, 3, H, W]."""
    img = torch.as_tensor(rgba)
    img = img[:, :, 3:4] * img[:, :, :3] + torch.ones(img.shape[0], img.shape[1], 3, dtype=img.dtype) * (1 - img[:, :, 3:4])
    return img.unsqueeze(0).permute(0, 3, 1, 2)


def composite(cov, paper):
    """synth's image [3, H, W] from the covered fraction [H, W] and the paper RGBA (torch, differentiable in paper): the
    pixel's RGBA is (1 - c) paper_rgb, c + (1 - c) paper_a."""
    c = torch.as_tensor(cov, dtype=torch.float64)
    P = torch.as_tensor(paper).to(torch.float64)
    rgba = torch.cat([(1 - c)[..., None] * P[:3], (c + (1 - c) * P[3])[..., None]], dim=-1)
    return synth_composite(rgba)[0]


def pixel_weights(cov, paper, g_img):
    """G [H, W] = sum_ch g_ch d out_ch / dc, and the paper's gradient [4] (the interior term)."""
    c = np.asarray(cov, dtype=np.float64)
    P = np.asarray(paper, dtype=np.float64)
    g = np.asarray(g_img, dtype=np.float64)
    u = 1 - c
    A = c + u * P[3]
    ia = 1 - P[3]
    G = sum(g[q] * (-P[q] * A + u * P[q] * ia - ia) for q in range(3))
    gp = np.array([np.sum(g[q] * u * A) for q in range(3)] + [np.sum(sum(g[q] * (u * u * P[q] - u) for q in range(3)))])
    return G, gp


def _line_intervals(o, d, caps, r):
    """(lo, hi, valid) per capsule: the parameters where o + s d lies strictly inside it (one interval: convex)."""
    A = d[0] ** 2 + d[1] ** 2
    lo = np.full(len(caps), np.inf)
    hi = np.full(len(caps), -np.inf)
    for e in (0, 2):
        qx, qy = o[0] - caps[:, e], o[1] - caps[:, e + 1]
        B = qx * d[0] + qy * d[1]
        disc = B * B - A * (qx * qx + qy * qy - r * r)
        ok = disc > 0
        sq = np.sqrt(np.where(ok, disc, 0.0))
        lo = np.where(ok, np.minimum(lo, (-B - sq) / A), lo)
        hi = np.where(ok, np.maximum(hi, (-B + sq) / A), hi)
    ex, ey = caps[:, 2] - caps[:, 0], caps[:, 3] - caps[:, 1]
    ll = ex * ex + ey * ey
    body = ll > 0
    ln = np.sqrt(np.where(body, ll, 1.0))
    mx, my = -ey / ln, ex / ln
    qx, qy = o[0] - caps[:, 0], o[1] - caps[:, 1]
    l, h = np.full(len(caps), -np.inf), np.full(len(caps), np.inf)
    for a0, a1, vlo, vhi in ((qx * ex + qy * ey, d[0] * ex + d[1] * ey, 0.0, ll),
                             (qx * mx + qy * my, d[0] * mx + d[1] * my, -r, r)):
        zero = a1 == 0
        inside = (a0 > vlo) & (a0 < vhi)
        a1s = np.where(zero, 1.0, a1)
        s0, s1 = (vlo - a0) / a1s, (vhi - a0) / a1s
        s0, s1 = np.where(a1 < 0, s1, s0), np.where(a1 < 0, s0, s1)
        l = np.where(zero, np.where(inside, l, np.inf), np.maximum(l, s0))
        h = np.where(zero, np.where(inside, h, -np.inf), np.minimum(h, s1))
    ok = body & (l < h)
    lo = np.where(ok, np.minimum(lo, l), lo)
    hi = np.where(ok, np.maximum(hi, h), hi)
    return lo, hi, lo < hi


def _visible_moments(lo, hi, s0, s1):
    """Integrals of 1 and s over [s0, s1] minus the union of the intervals (lo, hi)."""
    i0 = i1 = 0.0
    cur = s0
    while cur < s1:
        moved = True
        while moved:
            m = (lo <= cur) & (hi > cur)
            moved = bool(m.any())
            if moved:
                cur = float(hi[m].max())
        if cur >= s1:
            break
        ahead = lo[(lo > cur) & (lo < s1)]
        nx = float(ahead.min()) if ahead.size else s1
        i0 += nx - cur
        i1 += 0.5 * (nx - cur) * (nx + cur)
        cur = nx
    return i0, i1


def _unit(c):
    ex, ey = c[2] - c[0], c[3] - c[1]
    ln = math.hypot(ex, ey)
    return (ex / ln, ey / ln) if ln > 0 else (0.0, 0.0)


def capsule_gradients(sc, G):
    """[n_caps, 5]: d/d(ax, ay, bx, by, w) of sum_p G(p) c(p), the boundary integral of the module docstring."""
    H, W = sc.H, sc.W
    caps, cw = sc.caps, sc.cap_w
    out = np.zeros((len(caps), 5))
    phi = 2 * np.pi * (np.arange(ARC_NODES) + 0.5) / ARC_NODES
    U = np.stack([np.cos(phi), np.sin(phi)], axis=1)
    for c in range(len(caps)):
        a = caps[c]
        w = cw[c]
        others = np.arange(len(caps)) != c
        ex, ey = a[2] - a[0], a[3] - a[1]
        ln = math.hypot(ex, ey)
        if ln > 0:
            for sig in (1.0, -1.0):
                nx, ny = -ey / ln * sig, ex / ln * sig
                o = (a[0] + w * nx, a[1] + w * ny)
                d = (ex, ey)
                lo, hi, ok = _line_intervals(o, d, caps[others], cw[others])
                lo, hi = lo[ok], hi[ok]
                c0, c1 = 0.0, 1.0
                for p_, q_ in ((-ex, o[0]), (ex, W - o[0]), (-ey, o[1]), (ey, H - o[1])):
                    if p_ == 0:
                        if q_ < 0:
                            c0, c1 = 1.0, 0.0
                    elif p_ < 0:
                        c0 = max(c0, q_ / p_)
                    else:
                        c1 = min(c1, q_ / p_)
                if not c0 < c1:
                    continue
                # pixel pieces: the parameters where the line crosses a grid line
                cuts = [c0, c1]
                for v, dv, n in ((o[0], ex, W), (o[1], ey, H)):
                    if dv != 0:
                        k0, k1 = sorted(((v + c0 * dv), (v + c1 * dv)))
                        cuts += [(g - v) / dv for g in range(int(np.ceil(k0)), int(np.floor(k1)) + 1)]
                cuts = np.unique(np.clip(cuts, c0, c1))
                for s0, s1 in zip(cuts[:-1], cuts[1:]):
                    if s1 <= s0:
                        continue
                    m = 0.5 * (s0 + s1)
                    ix, iy = int(np.floor(o[0] + m * ex)), int(np.floor(o[1] + m * ey))
                    if not (0 <= ix < W and 0 <= iy < H) or G[iy, ix] == 0:
                        continue
                    i0, i1 = _visible_moments(lo, hi, s0, s1)
                    f = G[iy, ix] * ln
                    out[c, 0:2] += f * (i0 - i1) * np.array([nx, ny])
                    out[c, 2:4] += f * i1 * np.array([nx, ny])
                    out[c, 4] += f * i0
        e = np.array(_unit(a))
        prev = None if sc.first[c] else c - 1
        ep = np.zeros(2) if prev is None else np.array(_unit(caps[prev]))
        for end, (vx, vy) in ((False, (a[0], a[1])), (True, (a[2], a[3]))):
            if end and not sc.last[c]:
                continue
            de = U @ e
            keep = de >= 0 if end else (de <= 0) & (U @ ep >= 0)
            X = np.array([vx, vy]) + w * U
            keep &= (X[:, 0] >= 0) & (X[:, 0] < W) & (X[:, 1] >= 0) & (X[:, 1] < H)
            excl = np.ones(len(caps), dtype=bool)
            excl[c] = False
            if not end and prev is not None:
                excl[prev] = False
            for q in np.nonzero(excl)[0]:
                keep &= ~(_seg_dist(X[:, 0], X[:, 1], caps[q]) < cw[q])
            if not keep.any():
                continue
            ix = np.minimum(X[keep, 0].astype(np.int64), W - 1)
            iy = np.minimum(X[keep, 1].astype(np.int64), H - 1)
            f = G[iy, ix] * w * 2 * np.pi / ARC_NODES
            o_ = 2 if end else 0
            out[c, o_:o_ + 2] += (f[:, None] * U[keep]).sum(axis=0)
            out[c, 4] += f.sum()
    return out


def fold(sc, cap_grad):
    """Chain rule from the chords' endpoints and widths to the control points [N, 3L + 1, 2] and widths [N]."""
    N, L = sc.N, sc.L
    g = cap_grad.reshape(N, L, S, 5)
    Ba = bernstein(np.arange(S) / S)        # [4, S]
    Bb = bernstein(np.arange(1, S + 1) / S)
    gp = np.zeros((N, 3 * L + 1, 2))
    for j in range(L):
        gp[:, 3 * j:3 * j + 4] += np.einsum("ms,nsd->nmd", Ba, g[:, j, :, 0:2]) + np.einsum("ms,nsd->nmd", Bb, g[:, j, :, 2:4])
    return gp, g[..., 4].sum(axis=(1, 2))


def gradient(z, n_paths, n_segments, H, W, win, g_img, paper_trainable=True, caps=None):
    """d <synth(z), g_img> / dz (packed like z) at the forward whose sample winners are `win`."""
    sc = Scene(z, n_paths, n_segments, H, W, caps)
    G, gpaper = pixel_weights(coverage(win), sc.paper, g_img)
    gp, gw = fold(sc, capsule_gradients(sc, G))
    return np.concatenate([gp.reshape(-1), gw, gpaper if paper_trainable else np.zeros(4)])


def render(z, n_paths, n_segments, H, W, samples, win=None):
    """(image [3, H, W] float64 torch, winners [n, H, W])."""
    sc = Scene(z, n_paths, n_segments, H, W)
    if win is None:
        win = sc.winners(samples)
    return composite(coverage(win), sc.paper), win


class StrokeRender(torch.autograd.Function):
    """synth as an autograd Function: forward = render at the given samples, backward = the boundary gradient.  For
    ref_path.iterate: synth_fn = lambda z: StrokeRender.apply(z, meta)[None].float()."""

    @staticmethod
    def forward(ctx, z, meta):
        n_paths, n_segments, H, W, samples, paper_trainable = meta
        img, win = render(z.detach().cpu().numpy(), n_paths, n_segments, H, W, samples)
        ctx.meta, ctx.win, ctx.z = meta, win, z.detach().cpu().numpy()
        return img.to(z.device)

    @staticmethod
    def backward(ctx, g):
        n_paths, n_segments, H, W, _, paper_trainable = ctx.meta
        gz = gradient(ctx.z, n_paths, n_segments, H, W, ctx.win, g.detach().cpu().double().numpy(), paper_trainable)
        return torch.from_numpy(gz).to(g.device, g.dtype), None
