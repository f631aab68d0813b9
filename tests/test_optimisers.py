"""The `optimiser` setting on the CPU: which names apply_settings accepts, which drawers consult it and what engine calls
that issues (against a recording stand-in for the engine), the vdiff loop's switches between the chosen rule and Adam
against a transcription of the reference's train(), and the float64 oracle (oracle/optim_ref.py) against torch.optim."""
import json
import os

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from oracle import optim_ref as R
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import plugins as P

CHOSEN = ["AdamW", "Adagrad", "Adamax", "DiffGrad"]


class OptFake(FakeEngine):
    """FakeEngine plus set_optimizer and the latents of every drawer, so do_init runs for each of them."""

    def __init__(self, *, drawer=E.DRAWER_VQGAN, image_hw=(256, 256), grid=None, polygons=None, strokes=None, **kw):
        super().__init__(drawer=drawer, image_hw=image_hw, grid=grid or (1, 1), **kw)
        if drawer == E.DRAWER_SUPERRES:
            self.z_shape = (1, 3, image_hw[0] // 4, image_hw[1] // 4)
        elif drawer == E.DRAWER_POLYGON:
            self.z_shape = (len(polygons[1]) - 1, 4)
        elif drawer == E.DRAWER_STROKES:
            self.z_shape = (sum(E.stroke_z_layout(strokes[0], strokes[1])),)

    def set_optimizer(self, kind):
        self._log("set_optimizer", kind=kind)

    def set_synth_iteration(self, it):
        self._log("set_synth_iteration", it=it)


@pytest.fixture
def fake(monkeypatch, tmp_path):
    monkeypatch.setattr(api, "_engine_factory", OptFake)
    OptFake.loss_script = staticmethod(lambda it, n: np.full(n, 1.0 / (1 + it), dtype=np.float32))
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps({"ViT-B/16": [[0.1] * 512]}))
    monkeypatch.setenv("PIXRAY_ROOT", str(tmp_path))
    api.reset_settings()
    yield
    api.reset_settings()


def _drawer_settings(drawer, tmp_path):
    if drawer == "super_resolution":
        from PIL import Image
        rgb = (np.random.default_rng(4).random((32, 32, 3)) * 255).astype(np.uint8)
        Image.fromarray(rgb).save(tmp_path / "init.png")
        return dict(init_image=str(tmp_path / "init.png"), vector_prompts="none")
    if drawer == "vdiff":
        return dict(b200_weights={"vdiff": {"dummy": torch.zeros(1)}})
    if drawer == "fast_pixel":
        return dict(pixel_size=[8, 8])
    if drawer == "line_sketch":
        return dict(vector_prompts="none")
    return {}


def _init(tmp_path, drawer="vqgan", **kw):
    base = dict(prompts="x", drawer=drawer, size=[32, 32], clip_models="ViT-B/16", num_cuts=4, outdir="", seed="7",
                b200_allow_synthetic=True)
    base.update(_drawer_settings(drawer, tmp_path))
    base.update(kw)
    api.add_settings(**base)
    args = api.apply_settings()
    api.do_init(args)
    return args


@pytest.mark.parametrize("name", CHOSEN + ["Adam"])
def test_the_built_optimisers_pass_apply_settings(name):
    api.reset_settings()
    api.add_settings(prompts="x", optimiser=name)
    assert api.apply_settings().optimiser == name
    api.reset_settings()


@pytest.mark.parametrize("name,reason", [("AdamP", "per-slice projection"), ("SGD", "hot path")])
def test_adamp_and_unknown_names_stay_refused(name, reason):
    api.reset_settings()
    api.add_settings(prompts="x", optimiser=name)
    with pytest.raises(NotImplementedError, match=reason):
        api.apply_settings()
    api.reset_settings()


CONSULTING = ["vqgan", "fast_pixel", "super_resolution", "vdiff"]  # get_opts() is None (pixray.py:524-553)
OWN_ADAM = ["fft", "pixel", "line_sketch"]


@pytest.mark.parametrize("drawer", CONSULTING + OWN_ADAM)
def test_do_init_switches_the_rule_only_where_the_reference_consults_the_setting(fake, tmp_path, drawer):
    _init(tmp_path, drawer, optimiser="DiffGrad", iterations=5)
    calls = [c for c in api._state.engine.calls if c[0] == "set_optimizer"]
    if drawer in CONSULTING:
        assert calls == [("set_optimizer", {"kind": E.OPT_DIFFGRAD})]
        assert "reset_optimizer" not in api._state.engine.names()
    else:
        assert calls == [] and api._state.engine.names().count("reset_optimizer") == 1


@pytest.mark.parametrize("drawer", CONSULTING + OWN_ADAM)
def test_an_adam_session_issues_the_calls_it_issues_without_the_option(fake, tmp_path, drawer):
    args = _init(tmp_path, drawer, iterations=6, learning_rate_drops=[50])
    api.do_run(args)
    plain = list(api._state.engine.calls)
    api.reset_settings()
    args = _init(tmp_path, drawer, iterations=6, learning_rate_drops=[50], optimiser="Adam")
    api.do_run(args)
    assert api._state.engine.calls == plain and "set_optimizer" not in api._state.engine.names()


def _reference_vdiff_schedule(chosen, iterations, drops, max_loss_drops, learning_rate, sigmas, alphas):
    """pixray.py:1436-1512 with rebuild_optimisers (520-555) for the vdiff drawer, reduced to the optimiser objects: the
    (rule, lr) that takes the opt.step() of every iteration.  The losses keep improving, so only scheduled drops fire."""
    opt = (chosen, learning_rate)  # do_init -> rebuild_optimisers
    num_loss_drop, seq = 0, []
    for cur_it in range(iterations + 1):
        rebuild = False
        if cur_it < iterations:
            seq.append(opt)
            rebuild = cur_it in drops
        if cur_it >= 1:  # the vdiff block: a fresh optim.Adam at the schedule's step size
            opt = ("Adam", min(float(sigmas[cur_it] / alphas[cur_it]) * 0.001, 0.01))
        if cur_it == iterations:
            break
        if rebuild:
            num_loss_drop += 1
            if num_loss_drop > max_loss_drops:
                break
            opt = (chosen, learning_rate / 10 ** num_loss_drop)  # rebuild_optimisers
    return seq


def test_vdiff_host_loop_follows_the_reference_rule_switches(fake, tmp_path):
    args = _init(tmp_path, "vdiff", optimiser="DiffGrad", iterations=10, learning_rate_drops=[50])
    assert args.learning_rate_drops == [4] and not api._state.managed
    assert api.do_run(args) is True
    names = {v: k for k, v in E.OPTIMISERS.items()}
    kind, seq = E.OPT_ADAM, []
    for name, kw in api._state.engine.calls:
        if name == "set_optimizer":
            kind = kw["kind"]
        elif name == "iterate":
            seq.append((names[kind], kw["lr"]))
    d = api._state.drawer
    want = _reference_vdiff_schedule("DiffGrad", 10, [4], 1, 0.2, d.sigmas, d.alphas)
    assert [k for k, _ in seq] == [k for k, _ in want]
    assert [k for k, _ in want] == ["DiffGrad", "DiffGrad"] + ["Adam"] * 3 + ["DiffGrad"] + ["Adam"] * 4
    assert np.allclose([lr for _, lr in seq], [lr for _, lr in want], rtol=1e-6, atol=0)


def test_plugin_optimizer_takes_a_name(fake, tmp_path):
    _init(tmp_path, iterations=3)
    st = api._state
    eng = st.engine
    eng.calls.clear()
    P.Optimizer(st.session, st.drawer, 0.05, name="Adamax")
    P.Optimizer(st.session, st.drawer, 0.05, name="Adamax")
    P.Optimizer(st.session, st.drawer, 0.05)
    assert eng.calls == [("set_optimizer", {"kind": E.OPT_ADAMAX}), ("reset_optimizer", {}),
                         ("set_optimizer", {"kind": E.OPT_ADAM})]
    with pytest.raises(NotImplementedError):
        P.Optimizer(st.session, st.drawer, 0.05, name="AdamP")


# ------------------------------------------------------------------------------------------------------- the oracle
def _gradients(steps, n, seed):
    """Magnitudes from 1e-6 to 1e3, exact zeros and sign flips between consecutive steps."""
    rng = np.random.default_rng(seed)
    mag = 10.0 ** rng.uniform(-6, 3, size=(steps, n))
    sign = np.where(rng.random((steps, n)) < 0.5, -1.0, 1.0)
    g = mag * sign
    g[:, : n // 8] = 0.0
    g[1::2, n // 8: n // 4] = -g[0::2, n // 8: n // 4]  # steps is even
    g[rng.random((steps, n)) < 0.05] = 0.0
    return g


TORCH = {"Adam": torch.optim.Adam, "AdamW": torch.optim.AdamW, "Adagrad": torch.optim.Adagrad,
         "Adamax": torch.optim.Adamax}


@pytest.mark.parametrize("kind", sorted(TORCH))
def test_oracle_equals_torch_optim_across_a_reset(kind):
    n, steps, reset_at, lr = 256, 50, 25, 0.1
    g = _gradients(steps, n, 3)
    z0 = np.random.default_rng(5).normal(size=n)
    ref = R.Optimizer(kind, lr, n)
    z_ref = z0.copy()
    p = torch.nn.Parameter(torch.from_numpy(z0.copy()))
    opt = TORCH[kind]([p], lr=lr, foreach=False)
    for k in range(steps):
        if k == reset_at:
            ref.reset(lr / 10)
            opt = TORCH[kind]([p], lr=lr / 10, foreach=False)
        z_ref = ref.step(z_ref, g[k])
        p.grad = torch.from_numpy(g[k].copy())
        opt.step()
        assert np.abs(z_ref - p.detach().numpy()).max() <= 1e-12 * max(1.0, np.abs(z_ref).max()), (kind, k)


def test_oracle_diffgrad_first_two_steps_by_hand():
    lr, b1, b2, eps = 0.5, 0.9, 0.999, 1e-8
    z0, g1, g2 = np.array([0.3, -1.0, 2.0]), np.array([0.2, 0.0, -4.0]), np.array([-0.1, 0.5, -4.0])
    ref = R.Optimizer("DiffGrad", lr, 3)
    z1 = ref.step(z0, g1)
    z2 = ref.step(z1, g2)
    m1, v1 = 0.1 * g1, 0.001 * g1 ** 2
    xi1 = 1 / (1 + np.exp(-np.abs(0 - g1)))
    want1 = z0 - lr * np.sqrt(1 - b2) / (1 - b1) * (m1 * xi1) / (np.sqrt(v1) + eps)
    m2, v2 = b1 * m1 + 0.1 * g2, b2 * v1 + 0.001 * g2 ** 2
    xi2 = 1 / (1 + np.exp(-np.abs(g1 - g2)))
    want2 = want1 - lr * np.sqrt(1 - b2 ** 2) / (1 - b1 ** 2) * (m2 * xi2) / (np.sqrt(v2) + eps)
    assert np.allclose(z1, want1, rtol=0, atol=1e-15) and np.allclose(z2, want2, rtol=0, atol=1e-15)
    assert xi2[2] == 0.5  # equal consecutive gradients: friction 1/2
