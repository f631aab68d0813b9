"""Perceptors of different input resolutions in one session, on the host side: the cutout sets the engine is asked for
(the reference's cutoutsTable, pixray.py:642-649), the presets that need them (quality "best" and "supreme",
pixray.py:1824-1878), the refusal of spot prompts across resolutions, and the loss-vector layout of the cutout-space
losses (one entry per set, pixray.py:1392-1398).  A recording stand-in declares the capability; the plain stand-ins keep
today's refusals (tests/test_resnet_perceptor.py)."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from oracle import multires_ref as MR
from oracle import ref_path as R
from pixray_b200 import api
from pixray_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class MultiresFakeEngine(FakeEngine):
    TOWERS = E.B200Engine.TOWERS
    MAX_PERCEPTORS = E.B200Engine.MAX_PERCEPTORS
    MIXED_RESOLUTIONS = E.B200Engine.MIXED_RESOLUTIONS

    def __init__(self, **kw):
        super().__init__(**kw)
        self.cut_sets, self.set_of = E.cutout_sets(self.cut_size, [c["image_res"] for c in self.kw["clip"]])

    def num_losses(self):
        return super().num_losses() + sum(E.aux_loss_width(k, len(self.cut_sets)) - 1 for (k, _, _) in self.aux)

    def add_aux_loss(self, kind, weight, params):  # the first of its entries, as B200Engine.add_aux_loss returns
        super().add_aux_loss(kind, weight, params)
        return self.num_losses() - E.aux_loss_width(kind, len(self.cut_sets))


@pytest.fixture
def mfake(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", MultiresFakeEngine)
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "none.json").write_text(json.dumps({}))
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(size=[64, 64], num_cuts=8, outdir="", seed="7", b200_allow_synthetic=True, vector_prompts="none")
    base.update(kw)
    api.add_settings(**base)
    return api.do_init(api.apply_settings())


def test_cutout_sets_follow_first_appearance():
    assert E.cutout_sets(288, [288, 224, 224]) == ([288, 224], [0, 1, 1])
    assert E.cutout_sets(224, [224, 336, 224, 288]) == ([224, 336, 288], [0, 1, 0, 2])
    assert E.cutout_sets(224, [224, 224]) == ([224], [0, 0])


def test_quality_best_gives_two_sets(mfake, tmp_path):
    _init(tmp_path, prompts="a cat", quality="best")
    eng = api._state.engine
    assert [c["image_res"] for c in eng.kw["clip"]] == [288, 224, 224]
    assert [c["out_dim"] for c in eng.kw["clip"]] == [640, 512, 512]
    assert eng.cut_size == 288 and eng.cut_sets == [288, 224] and eng.set_of == [0, 1, 1]
    assert list(api._state.cutouts_table) == [288, 224]
    assert [m.cut_set for m in api._state.cutouts_table.values()] == [0, 1]
    assert api._state.make_cutouts is api._state.cutouts_table[288]
    assert [p.input_resolution for p in api._state.perceptors] == [288, 224, 224]
    assert ("set_batches", {"batches": 2}) in eng.calls


def test_quality_supreme_gives_four_perceptors(mfake, tmp_path):
    _init(tmp_path, prompts="a cat", quality="supreme")
    eng = api._state.engine
    assert len(eng.kw["clip"]) == 4 and eng.cut_sets == [288, 224] and eng.set_of == [0, 1, 1, 1]
    assert set(eng.modules) == {E.MOD_VQGAN, E.MOD_CLIP0, E.MOD_CLIP1, E.MOD_CLIP2, E.MOD_CLIP3}
    assert (E.MOD_CLIP0, E.MOD_CLIP3) == (1, 4)
    assert sorted(eng.prompts) == [0, 1, 2, 3]


@pytest.mark.parametrize("models,sets", [("ViT-L/14@336px,ViT-B/16", [336, 224]), ("ViT-B/16,ViT-L/14@336px", [224, 336])])
def test_vit_l336_beside_a_224_pixel_tower_in_either_order(mfake, tmp_path, models, sets):
    _init(tmp_path, prompts="a cat", clip_models=models)
    eng = api._state.engine
    assert eng.cut_size == sets[0] and eng.cut_sets == sets
    assert list(api._state.cutouts_table) == sets


def test_spot_prompts_across_resolutions_are_refused(mfake, tmp_path):
    with pytest.raises(ValueError, match=r"pixray.py:1270-1276.*slip.py:53-57"):
        _init(tmp_path, prompts="a cat", quality="best", spot_prompts="a dog")


def test_spot_prompts_with_one_resolution_are_not_refused(mfake, tmp_path):
    mask = np.ones((3, 224, 224), dtype=bool)
    _init(tmp_path, prompts="a cat", clip_models="ViT-B/32,ViT-B/16", spot_prompts="a dog", spot_file=mask)
    assert "set_spot_prompts" in api._state.engine.names()


def test_five_perceptors_are_refused(mfake, tmp_path):
    with pytest.raises(NotImplementedError, match="at most 4 perceptors"):
        _init(tmp_path, prompts="a cat", clip_models="RN50x4,RN101,ViT-B/32,ViT-B/16,RN50")


def test_loss_vector_layout_with_cutout_space_losses(mfake, tmp_path):
    _init(tmp_path, prompts="a cat", quality="best", custom_loss="saturation,symmetry,palette,smoothness",
          palette="#000000;#ffffff")
    st = api._state
    eng = st.engine
    # three perceptors with one text prompt each, then saturation x 2 sets, symmetry, palette x 2, smoothness x 2
    assert eng.num_losses() == 3 + 2 + 1 + 2 + 2
    idx = [t["loss"]._index for t in st.custom]
    assert idx == [3, 5, 6, 8]
    vec = np.arange(eng.num_losses(), dtype=np.float32)
    eng.read_losses = lambda: vec
    got = [t["loss"].get_loss(None, None, None) for t in st.custom]
    assert [float(x) for x in got[0]] == [3.0, 4.0]
    assert float(got[1]) == 5.0
    assert [float(x) for x in got[2]] == [6.0, 7.0] and [float(x) for x in got[3]] == [8.0, 9.0]


def test_one_resolution_keeps_scalar_losses(mfake, tmp_path):
    _init(tmp_path, prompts="a cat", clip_models="ViT-B/32,ViT-B/16", custom_loss="saturation")
    loss = api._state.custom[0]["loss"]
    api._state.engine.read_losses = lambda: np.array([1.0, 2.0, 7.0], dtype=np.float32)
    assert isinstance(loss.get_loss(None, None, None), torch.Tensor) and float(loss.get_loss(None, None, None)) == 7.0


def test_train_iteration_cuts_every_resolution_and_clears_the_cache():
    from pixray_b200 import plugins as P

    class Rec:
        def __init__(self, cs):
            self.cs, self.transforms, self.seen = cs, "cached", []

        def __call__(self, out):
            self.seen.append(out)
            return f"cut{self.cs}"

    class Perc:
        def __init__(self, res, log):
            self.input_resolution, self.log = res, log

        def encode_image(self, x):
            self.log.append((self.input_resolution, x))
            return torch.zeros(1)

    class Sess:
        cur_iteration = 0

        def backward(self, drawer):
            pass

    class Drawer:
        def synth(self, it):
            return "img"

        def clip_z(self):
            pass

    class Opt:
        def zero_grad(self):
            pass

        def step(self):
            pass

    log = []
    table = {288: Rec(288), 224: Rec(224)}
    percs = [Perc(288, log), Perc(224, log), Perc(224, log)]
    P.train_iteration(Sess(), Drawer(), table, percs, [[], [], []], Opt())
    assert log == [(288, "cut288"), (224, "cut224"), (224, "cut224")]
    assert all(m.seen == ["img"] and m.transforms is None for m in table.values())


def test_cutout_kernel_has_no_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "pixray_b200", "csrc", "kernels_cutouts.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stderr.splitlines()
    fwd = [i for i, l in enumerate(lines) if "Compiling entry function" in l and "cutout_fwd_kernel" in l]
    assert fwd
    for i in fwd:
        info = next(l for l in lines[i + 1:i + 6] if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in info, info


def test_oracle_reproduces_the_reference_ascend_txt():
    """oracle/multires_ref.iterate_sets against the unmodified reference ascend_txt with two MakeCutouts
    (tests/golden/multires_ascend.npz, oracle/make_golden_multires.py)."""
    from oracle.make_golden_multires import ASPECT, MODELS, SIZES

    G = np.load(os.path.join(ROOT, "tests", "golden", "multires_ascend.npz"))
    sets = [dict(cs=cs, transforms=torch.from_numpy(G[f"T{cs}"])) for cs in SIZES]
    percs, prompts = [], []
    for name, (res, patch, width, layers, heads, dim, seed) in MODELS.items():
        percs.append((R.init_clip_weights(R.ClipVisual(res, patch, width, layers, heads, dim), seed), SIZES.index(res)))
        pe = torch.from_numpy(G[f"pe_{name}"])
        prompts.append([(pe[0:1], 1.0, float("-inf")), (pe[1:2], -0.4, float("-inf"))])
    palette = G["palette"]
    w = G["loss_weights"]
    aux = [(float(w[0]), "cutouts", lambda b: R.saturation_loss(b, 1.3)),
           (float(w[1]), "cutouts", lambda b: R.palette_loss(b, palette, 0.8)[0]),
           (float(w[2]), "cutouts", lambda b: R.smoothness_loss(b, 0.9))]
    ref = MR.iterate_sets(torch.from_numpy(G["out"]), sets, percs, prompts,
                          image_prompts=[(torch.from_numpy(G["timg"]), 0.7)], aux=aux, zoom_padding=str(G["zoom_padding"]),
                          fill=float(G["fill"]), aspect=ASPECT)
    got = np.array([float(x) for x in ref["losses"]], dtype=np.float32)
    assert got.shape == G["losses"].shape == (3 * 3 + 3 * 2,)
    assert np.abs(got - G["losses"]).max() <= 1e-6
    # SmoothnessLoss takes sqrt(0) on the constant fill of the wide cutouts: the reference's own gradient is NaN there,
    # and the oracle's must be NaN at exactly the same pixels
    d, ok = ref["image_grad"].numpy(), np.isfinite(G["d_out"])
    assert np.array_equal(np.isfinite(d), ok) and ok.mean() > 0.5
    assert np.abs(d[ok] - G["d_out"][ok]).max() <= 1e-6 * max(1.0, np.abs(G["d_out"][ok]).max())


def test_a_batch_of_another_set_size_is_refused():
    """B200Engine.encode_image checks the batch against the perceptor's own cutout set before the engine copies it."""
    from types import SimpleNamespace
    eng = SimpleNamespace(cut_sets=[224, 336], set_of=[0, 1], n_local=4, clip_dims=[512, 768],
                          _new=lambda *shape: torch.zeros(shape))
    with pytest.raises(E.EngineError, match="336 x 336 cutouts"):
        E.B200Engine.encode_image(eng, 1, torch.zeros(4, 3, 224, 224))
    with pytest.raises(E.EngineError, match="224 x 224 cutouts"):
        E.B200Engine.encode_image(eng, 0, torch.zeros(4, 3, 336, 336))


def test_train_iteration_refuses_one_make_cutouts_for_two_resolutions():
    from types import SimpleNamespace
    from pixray_b200 import plugins as P
    mc = SimpleNamespace(cut_size=224)
    percs = [SimpleNamespace(input_resolution=224), SimpleNamespace(input_resolution=336)]
    with pytest.raises(ValueError, match="input resolution 336"):
        P.train_iteration(None, None, mc, percs, [[], []], None)
