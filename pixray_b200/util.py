"""Settings helpers whose behaviour the reference's own unit tests pin (tests/test_util.py, tests/test_pixray.py):
unit strings like "200 iterations" / "50%", pipe-separated lists, output file paths.  Semantics follow
util.py:32-36, 49-71 and pixray.py:1430-1433, 1999-2003; written from those behaviours, not copied."""
import re
from pathlib import PurePath

_NUM = r"\d*\.?\d+"
_ITER_UNITS = ("i", "iter", "iterations")
_PCT_UNITS = ("p", "%", "percent")


def get_file_path(directory, filename, suffix):
    """util.py:32-36: join, force the suffix, reject empty names and names containing a path separator."""
    if filename is None:
        raise ValueError("Invalid filename specified.")
    name = filename.strip()
    if name == "" or "/" in name or "\\" in name:
        raise ValueError("Invalid filename specified.")
    return str(PurePath(directory, filename).with_suffix(suffix))


def parse_unit(value, total_iterations, argument_name, default_unit="%"):
    """util.py:49-65: "<number>[ ]<unit>" -> iteration count; bare numbers take `default_unit`; percentages are of
    `total_iterations`; truncation toward zero."""
    if value is None:
        return None
    text = str(value).lower().strip()
    m = re.fullmatch(rf"({_NUM})\s*([a-z%]*)", text)
    if m:
        number, unit = float(m.group(1)), m.group(2) or default_unit
        if unit in _ITER_UNITS:
            return int(number)
        if unit in _PCT_UNITS:
            return int(number * 0.01 * total_iterations)
    raise ValueError(f"Invalid value for {argument_name}, please use a digit-unit combination like "
                     "'20 iterations' or '50%'.")


def split_pipes(attribute):
    """util.py:67-71: falsy values pass through, otherwise split on '|' and strip."""
    if not attribute:
        return attribute
    return [part.strip() for part in attribute.split("|")]


def get_learning_rate_drops(learning_rate_drops, iterations):
    """pixray.py:1999-2003: percentages of (iterations - 1)."""
    if learning_rate_drops is None:
        return []
    return [parse_unit(n, iterations - 1, "learning_rate_drops") for n in learning_rate_drops]


def apply_overlay(args, cur_it):
    """pixray.py:1430-1433."""
    return (args.overlay_image is not None and (cur_it % args.overlay_every) == args.overlay_offset
            and (args.overlay_until is None or cur_it < args.overlay_until))


def vdiff_schedule(iterations, vdiff_skip=0.0):
    """VdiffDrawer.init_from_tensor's default schedule (vdiff.py:113-126): t = linspace(top, 0, iterations + 2)[:-1] through
    the spliced DDPM / cosine schedule (diffusion/utils.py:63-78), then alpha = cos(pi t / 2), sigma = sin(pi t / 2)
    (utils.py:52-55).  Returns float32 numpy arrays (steps, alphas, sigmas) of length iterations + 1."""
    import numpy as np
    top = 1.0 - vdiff_skip / 100.0  # util.map_number(vdiff_skip, 0, 100, 1, 0)
    t = np.linspace(top, 0.0, iterations + 2, dtype=np.float32)[:-1].astype(np.float64)
    ddpm_crossover, cosine_crossover = 0.48536712, 0.80074257
    big_t = t * (1 + cosine_crossover - ddpm_crossover)
    ddpm_t = big_t + ddpm_crossover - cosine_crossover
    log_snr = -np.log(np.expm1(1e-4 + 10 * ddpm_t ** 2))
    alpha, sigma = np.sqrt(1 / (1 + np.exp(-log_snr))), np.sqrt(1 / (1 + np.exp(log_snr)))
    ddpm_part = np.arctan2(sigma, alpha) / np.pi * 2
    steps = np.where(big_t < cosine_crossover, big_t, ddpm_part)
    return (steps.astype(np.float32), np.cos(steps * np.pi / 2).astype(np.float32),
            np.sin(steps * np.pi / 2).astype(np.float32))


VDIFF_ROUNDUP = 128  # vdiff.py ROUNDUP_SIZE


def vdiff_gen_size(width, height):
    """VdiffDrawer's U-Net size for a canvas (vdiff.py:55-58, 165-170): gen = ceil(side / 128) * 128 per side, margins
    int((gen - canvas) / 2).  Returns (gen_w, gen_h, margin_x, margin_y).  The image is pixels[:, :, my:my+H, mx:mx+W],
    except when both margins are zero (each side 0 or 1 pixel short of a multiple of 128): the reference does not
    crop then, and the image is the whole gen-size frame (vdiff_image_size)."""
    gw = -(-int(width) // VDIFF_ROUNDUP) * VDIFF_ROUNDUP
    gh = -(-int(height) // VDIFF_ROUNDUP) * VDIFF_ROUNDUP
    return gw, gh, (gw - int(width)) // 2, (gh - int(height)) // 2


def vdiff_image_size(width, height):
    """(width, height) of the image VdiffDrawer.synth returns for a canvas: the canvas, or the gen size when no margin
    is cut (vdiff.py:167-168)."""
    gw, gh, mx, my = vdiff_gen_size(width, height)
    return (int(width), int(height)) if (mx or my) else (gw, gh)


# ------------------------------------------------------------------------------------------------ init images (host, init time)
def _perlin_2d(rng, shape, res):
    """perlin_numpy.generate_perlin_noise_2d [UPSTREAM pvigier/perlin-numpy, un-vendored; requirements.txt]: gradient noise
    on a res[0] x res[1] lattice, quintic interpolant, scaled by sqrt(2)."""
    import numpy as np
    delta = (res[0] / shape[0], res[1] / shape[1])
    d = (shape[0] // res[0], shape[1] // res[1])
    grid = np.mgrid[0:res[0]:delta[0], 0:res[1]:delta[1]].transpose(1, 2, 0) % 1
    angles = 2 * np.pi * rng.random((res[0] + 1, res[1] + 1))
    gradients = np.dstack((np.cos(angles), np.sin(angles))).repeat(d[0], 0).repeat(d[1], 1)
    g00, g10 = gradients[:-d[0], :-d[1]], gradients[d[0]:, :-d[1]]
    g01, g11 = gradients[:-d[0], d[1]:], gradients[d[0]:, d[1]:]
    n00 = np.sum(np.dstack((grid[:, :, 0], grid[:, :, 1])) * g00, 2)
    n10 = np.sum(np.dstack((grid[:, :, 0] - 1, grid[:, :, 1])) * g10, 2)
    n01 = np.sum(np.dstack((grid[:, :, 0], grid[:, :, 1] - 1)) * g01, 2)
    n11 = np.sum(np.dstack((grid[:, :, 0] - 1, grid[:, :, 1] - 1)) * g11, 2)
    t = grid * grid * grid * (grid * (grid * 6 - 15) + 10)
    n0 = n00 * (1 - t[:, :, 0]) + t[:, :, 0] * n10
    n1 = n01 * (1 - t[:, :, 0]) + t[:, :, 0] * n11
    return np.sqrt(2) * ((1 - t[:, :, 1]) * n0 + t[:, :, 1] * n1)


def fractal_noise_2d(rng, shape, res, octaves):
    """perlin_numpy.generate_fractal_noise_2d (persistence 0.5, lacunarity 2)."""
    import numpy as np
    noise, frequency, amplitude = np.zeros(shape), 1, 1.0
    for _ in range(octaves):
        noise += amplitude * _perlin_2d(rng, shape, (frequency * res[0], frequency * res[1]))
        frequency *= 2
        amplitude *= 0.5
    return noise


def random_noise_image(w, h, rng=None):
    """pixray.py:207-224 (`init_noise='pixels'`, the reference's DEFAULT start image): three fractal-noise channels,
    normalised, pushed through contrast_noise.  Returns uint8 [h, w, 3]."""
    import numpy as np
    rng = rng or np.random.default_rng()
    if w > 1024 or h > 1024:
        side, octp = 2048, 6
    elif w > 512 or h > 512:
        side, octp = 1024, 5
    elif w > 256 or h > 256:
        side, octp = 512, 4
    else:
        side, octp = 256, 3

    def chan():
        n = fractal_noise_2d(rng, (side, side), (32, 32), octp)
        n = (n - n.min()) / (n.max() - n.min())                 # NormalizeData
        n = 0.9998 * n + 0.0001                                 # contrast_noise
        return 1 / (1 + np.power(n / (1 - n), -2))

    stack = np.dstack((chan(), chan(), chan()))
    return (255.999 * stack[:h, :w, :]).astype("uint8")


def random_gradient_image(w, h, rng=None):
    """pixray.py:239-242 (`init_noise='gradient'`).  Returns uint8 [h, w, 3]."""
    import numpy as np
    rng = rng or np.random.default_rng()
    start = (0, 0, int(rng.integers(0, 255)))
    stop = (int(rng.integers(1, 255)), int(rng.integers(2, 255)), int(rng.integers(3, 128)))
    horizontal = (True, False, False)
    out = np.zeros((h, w, 3), dtype=float)
    for i, (a, b, hz) in enumerate(zip(start, stop, horizontal)):
        out[:, :, i] = np.tile(np.linspace(a, b, w), (h, 1)) if hz else np.tile(np.linspace(a, b, h), (w, 1)).T
    return np.uint8(out)
