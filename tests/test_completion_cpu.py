"""CPU: shape completion (`--mode=eval_completion`) -- the metric oracle on hand-built clouds, reading make_partial's index,
planning the packed sampling calls, the pair list of one `mdb_chamfer_pairs` launch, every refused configuration and the
command line."""
import json
import math
import os

import numpy as np
import pytest

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from meshdiffusion_b200.diffusion import completion
from oracle import completion_oracle as co


def _cloud(n, seed):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (n, 3)).astype(np.float32)


# ---- oracle ------------------------------------------------------------------------------------------------------
def test_oracle_translate_gives_uhd_of_the_shift():
    # points 10 apart and a shift of about 1.1: every x's nearest y is its own translate
    x = (10.0 * np.stack(np.meshgrid(*[np.arange(4)] * 3), -1).reshape(-1, 3) + _cloud(64, 0)).astype(np.float32)
    d = np.array([0.25, -0.5, 1.0], np.float64)
    y = (x.astype(np.float64) + d).astype(np.float32)
    assert math.isclose(co.uhd(x, y), np.linalg.norm(d), rel_tol=1e-5)
    cd, mean_ab, max_ab = co.pair_distances(x, y)
    assert math.isclose(math.sqrt(max_ab), co.uhd(x, y), rel_tol=1e-12)
    assert math.isclose(mean_ab, float(np.dot(d, d)), rel_tol=1e-5) and math.isclose(cd, 2 * mean_ab, rel_tol=1e-5)


def test_oracle_subset_partial_gives_zero_uhd():
    c = _cloud(200, 1)
    assert co.uhd(c[::3], c) == 0.0
    assert co.pair_distances(c[::3], c)[1:] == (0.0, 0.0)
    assert co.uhd(c, c[::3]) > 0  # one-sided


def test_oracle_identical_completions_give_zero_tmd():
    c = _cloud(100, 2)
    assert co.tmd([c, c.copy(), c.copy()]) == 0.0
    assert co.tmd([c, _cloud(100, 3)]) == pytest.approx(2.0 * co.chamfer(c, _cloud(100, 3)))
    lo, mean = co.accuracy([c, _cloud(100, 3)], c)
    assert lo == 0.0 and mean == pytest.approx(co.chamfer(_cloud(100, 3), c) / 2)


def test_oracle_sign_agreement_and_visible_faces():
    assert co.sign_agreement([0.5, -0.2, 0.1, -1.0], [1, 1, 1, -1], [1, 1, 0, 1]) == pytest.approx(2 / 3)
    assert math.isnan(co.sign_agreement([1.0], [1], [0]))
    assert co.visible_face_ids(np.array([[-1, 4, 4], [2, -1, 0]])) == [0, 2, 4]


# ---- index -------------------------------------------------------------------------------------------------------
SETTINGS = {"resolution": 64, "views": [0, 17], "res": 256, "mesh_scale": 1.1, "deform_scale": 3.0}


def _entry(shape, view, source=None):
    return {"file": f"{shape:06d}_view{view:02d}.pt", "shape": shape, "view": view,
            "source": source or f"/data/grid_{shape}.pt", "mvp": np.eye(4).tolist(), "res": 256}


def _write_index(d, name, entries, touch=True, **over):
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "w") as fh:
        json.dump({**SETTINGS, **over, "files": entries}, fh)
    if touch:
        for e in entries:
            open(os.path.join(d, e["file"]), "wb").close()


def test_read_single_index_sorted(tmp_path):
    d = str(tmp_path / "partial")
    _write_index(d, "index.json", [_entry(1, 0), _entry(0, 17), _entry(0, 0)])
    settings, entries = completion.read_index(d)
    assert settings == {"resolution": 64, "res": 256, "mesh_scale": 1.1, "deform_scale": 3.0}
    assert [(e["shape"], e["view"]) for e in entries] == [(0, 0), (0, 17), (1, 0)]


def test_read_per_rank_union(tmp_path):
    d = str(tmp_path / "partial")
    _write_index(d, "index_0.json", [_entry(0, 0), _entry(2, 0)])
    _write_index(d, "index_1.json", [_entry(1, 0), _entry(3, 0)])
    _, entries = completion.read_index(d)
    assert [e["shape"] for e in entries] == [0, 1, 2, 3]
    _write_index(d, "index_2.json", [_entry(4, 0)], deform_scale=1.5)
    with pytest.raises(ValueError, match="made with"):
        completion.read_index(d)


def test_read_index_refusals(tmp_path):
    d = str(tmp_path / "partial")
    with pytest.raises(FileNotFoundError, match="make_partial"):
        completion.read_index(d)
    _write_index(d, "index.json", [_entry(0, 0), _entry(1, 0)], touch=False)
    open(os.path.join(d, _entry(0, 0)["file"]), "wb").close()
    with pytest.raises(FileNotFoundError, match="000001_view00.pt"):
        completion.read_index(d)
    _write_index(d, "index.json", [])
    with pytest.raises(ValueError, match="no files"):
        completion.read_index(d)
    _write_index(d, "index.json", [_entry(0, 0), _entry(0, 0)])
    with pytest.raises(ValueError, match="twice"):
        completion.read_index(d)


def test_source_mismatch_is_refused():
    entries = [_entry(0, 0, "/a/grid_0.pt"), _entry(1, 0, "/a/grid_1.pt")]
    completion.check_sources(entries, ["/a/grid_0.pt\n", "/a/grid_1.pt"])
    with pytest.raises(ValueError, match="was made from"):
        completion.check_sources(entries, ["/a/grid_0.pt", "/b/grid_1.pt"])
    with pytest.raises(ValueError, match="selects 1"):
        completion.check_sources(entries, ["/a/grid_0.pt"])


# ---- planning ----------------------------------------------------------------------------------------------------
def test_plan_calls_packs_and_pads():
    assert completion.partials_per_call(8, 2) == 4 and completion.partials_per_call(10, 10) == 1
    calls = completion.plan_calls([1, 3, 5, 7, 9, 11], 4)
    assert calls == [([1, 3, 5, 7], 4), ([9, 11, 11, 11], 2)]
    assert completion.plan_calls([0, 1, 2, 3], 2) == [([0, 1], 2), ([2, 3], 2)]
    assert completion.plan_calls([], 3) == []


def test_group_pairs_layout():
    n, k = 2, 3
    ok = [True] * 6
    pairs, roles = completion.group_pairs(n, k, [True, True], ok)
    assert len(pairs) == n * (k + k * (k - 1) // 2 + k)
    comp = lambda i, j: 2 * n + i * k + j  # noqa: E731
    assert pairs[:3] == [(comp(0, 0), 0), (comp(0, 1), 0), (comp(0, 2), 0)]
    assert pairs[3:6] == [(comp(0, 0), comp(0, 1)), (comp(0, 0), comp(0, 2)), (comp(0, 1), comp(0, 2))]
    assert pairs[6:9] == [(2, comp(0, j)) for j in range(3)]
    assert roles[9] == (1, "gt", 0) and all(a != b for a, b in pairs)
    # an empty completion and an unscored partial drop their pairs
    pairs, roles = completion.group_pairs(n, k, [False, True], [True, True, True, True, False, True])
    assert all(r[0] == 1 for r in roles) and len(pairs) == 2 + 1 + 2
    assert not any(comp(1, 1) in p for p in pairs)


# ---- driver refusals and command line -----------------------------------------------------------------------------
def _config(tmp_path, **eval_kw):
    from configs import res64
    cfg = res64.get_config()
    cfg.device = "cpu"
    cfg.eval.eval_dir = str(tmp_path / "out")
    cfg.eval.ckpt_path = str(tmp_path / "missing.pth")
    cfg.eval.batch_size = 4
    cfg.eval.completion_k = 2
    cfg.sampling.method = "dpm_solver"
    from meshdiffusion_b200.geometry import dmtet
    cfg.eval.tet_path = dmtet.tet_grid_path(64)
    for k, v in eval_kw.items():
        cfg.eval[k] = v
    return cfg


@pytest.fixture
def no_model(monkeypatch):
    """Fails the test if the driver gets as far as building a network."""
    def refuse(config):
        raise AssertionError("the driver built a model before checking its arguments")
    monkeypatch.setattr(completion, "_setup", refuse)
    return completion


def _dataset(tmp_path, cfg, n=2):
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps([f"/data/grid_{i}.pt" for i in range(n)]))
    cfg.data.meta_path = str(meta)
    _write_index(str(tmp_path / "out" / "partial"), "index.json", [_entry(i, 0) for i in range(n)])


@pytest.mark.parametrize("case", ["k_one", "k_not_int", "batch_not_multiple", "batch_below_k", "pc_packed", "ddim",
                                  "unknown_sampler", "empty_index", "source_mismatch", "resolution", "no_tet_path"])
def test_driver_refuses(tmp_path, no_model, case):
    cfg = _config(tmp_path)
    _dataset(tmp_path, cfg)
    if case == "k_one":
        cfg.eval.completion_k = 1
    elif case == "k_not_int":
        cfg.eval.completion_k = 2.5
    elif case == "batch_not_multiple":
        cfg.eval.batch_size = 5
    elif case == "batch_below_k":
        cfg.eval.completion_k = 8
    elif case == "pc_packed":
        cfg.sampling.method = "pc"
    elif case == "ddim":
        cfg.sampling.method = "ddim"
    elif case == "unknown_sampler":
        cfg.sampling.method = "euler"
    elif case == "empty_index":
        _write_index(str(tmp_path / "out" / "partial"), "index.json", [])
    elif case == "source_mismatch":
        (tmp_path / "list.json").write_text(json.dumps(["/data/grid_0.pt", "/other/grid_1.pt"]))
    elif case == "resolution":
        _write_index(str(tmp_path / "out" / "partial"), "index.json", [_entry(0, 0)], resolution=128)
    elif case == "no_tet_path":
        cfg.eval.tet_path = "PLACEHOLDER"
    with pytest.raises((ValueError, FileNotFoundError)) as e:
        no_model.eval_completion(cfg)
    if case == "pc_packed":
        assert "first partial" in str(e.value)


def test_driver_accepts_valid_arguments_up_to_the_model(tmp_path, no_model):
    for method, batch in (("dpm_solver", 4), ("dpm_solver", 2), ("pc", 2)):
        cfg = _config(tmp_path)
        _dataset(tmp_path, cfg)
        cfg.sampling.method = method
        cfg.eval.batch_size = batch
        with pytest.raises(AssertionError, match="built a model"):
            no_model.eval_completion(cfg)


def test_command_line_accepts_the_mode():
    import main_diffusion
    path, mode, overrides = main_diffusion.parse_args(
        ["--config=configs/res64.py", "--mode=eval_completion", "--config.eval.completion_k=4",
         "--config.eval.partial_dir=/tmp/p"])
    assert mode == "eval_completion" and path == "configs/res64.py"
    assert ("eval.completion_k", 4) in overrides and ("eval.partial_dir", "/tmp/p") in overrides
