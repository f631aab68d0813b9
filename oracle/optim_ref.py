"""float64 restatement of the five update rules args.optimiser picks (pixray.py:536-551) for the tests, each with the
constructor defaults pixray builds it with (only lr is passed):

    Adam      torch.optim.Adam      (betas 0.9 / 0.999, eps 1e-8)
    AdamW     torch.optim.AdamW     (same, weight_decay 0.01, applied to z before the Adam step)
    Adagrad   torch.optim.Adagrad   (eps 1e-10, lr_decay 0, initial_accumulator_value 0)
    Adamax    torch.optim.Adamax    (betas 0.9 / 0.999, eps 1e-8)
    DiffGrad  torch_optimizer 0.1.0 DiffGrad (betas 0.9 / 0.999, eps 1e-8, weight_decay 0)

The first four are checked against the installed torch.optim by the tests.  torch_optimizer is not vendored, so DiffGrad
is restated from its published 0.1.0 source; its parity with that package is not pinned by a test here.

An instance is one optimiser object of the reference: `step` applies one update to z (clip_z is the caller's), `reset`
is rebuild_optimisers building a fresh one (state 0, t = 0).  Pure numpy.
"""
import numpy as np

KINDS = ("Adam", "AdamW", "Adagrad", "Adamax", "DiffGrad")
ADAMW_WEIGHT_DECAY = 0.01
ADAGRAD_EPS = 1e-10


class Optimizer:
    def __init__(self, kind, lr, n, betas=(0.9, 0.999), eps=1e-8):
        if kind not in KINDS:
            raise ValueError(f"unknown optimiser {kind!r}")
        self.kind, self.lr, self.n = kind, float(lr), int(n)
        self.b1, self.b2, self.eps = float(betas[0]), float(betas[1]), float(eps)
        self.reset()

    def reset(self, lr=None):
        """A fresh instance (rebuild_optimisers), optionally at a new learning rate."""
        if lr is not None:
            self.lr = float(lr)
        self.t = 0
        self.m = np.zeros(self.n)
        self.v = np.zeros(self.n)  # Adam / AdamW / DiffGrad: second moment; Adagrad: sum of g^2; Adamax: the inf norm u
        self.p = np.zeros(self.n)  # DiffGrad: the previous gradient

    def step(self, z, g, lr_scale=1.0):
        """z, g: float64 arrays of n; returns the updated z.  lr_scale multiplies lr (the line drawer's per-range rates)."""
        z = np.asarray(z, dtype=np.float64).reshape(-1)
        g = np.asarray(g, dtype=np.float64).reshape(-1)
        lr = self.lr * lr_scale
        b1, b2, eps = self.b1, self.b2, self.eps
        self.t += 1
        bc1, bc2 = 1.0 - b1 ** self.t, 1.0 - b2 ** self.t
        if self.kind == "Adagrad":
            self.v = self.v + g * g
            return z - lr * g / (np.sqrt(self.v) + ADAGRAD_EPS)
        if self.kind == "Adamax":
            self.m = b1 * self.m + (1 - b1) * g
            self.v = np.maximum(b2 * self.v, np.abs(g) + eps)
            return z - (lr / bc1) * self.m / self.v
        if self.kind == "AdamW":
            z = z * (1.0 - lr * ADAMW_WEIGHT_DECAY)
        self.m = b1 * self.m + (1 - b1) * g
        self.v = b2 * self.v + (1 - b2) * g * g
        if self.kind == "DiffGrad":
            xi = 1.0 / (1.0 + np.exp(-np.abs(self.p - g)))  # the friction coefficient dfc
            self.p = g.copy()
            return z - (lr * np.sqrt(bc2) / bc1) * (self.m * xi) / (np.sqrt(self.v) + eps)
        return z - (lr / bc1) * self.m / (np.sqrt(self.v) / np.sqrt(bc2) + eps)
