"""Training snapshots (learninghumanoidwalking_b200/rl/snapshot.py) without a GPU: the latest.json pointer, pruning of older
snapshots, and the loader's refusals (mixed iterations, world size, --num-procs, env, precision, format, missing files),
also through `run_experiment.py resume`, which must refuse before it writes anything."""
import argparse
import json
import pickle

import pytest
import torch

from learninghumanoidwalking_b200.rl import snapshot
from learninghumanoidwalking_b200.rl.snapshot import FORMAT, SnapshotError


def _fake(run_dir, itr=3, world=1, shard_itr=None, num_procs=64, env="jvrc_walk", precision=64, n_itr=10):
    """A snapshot with the metadata of a real one and tiny payloads."""
    root = snapshot.snapshot_root(run_dir)
    d = root / f"itr_{itr}"
    d.mkdir(parents=True, exist_ok=True)
    snapshot.save_file(dict(format=FORMAT, itr=itr, world=world, args=dict(num_procs=num_procs, n_itr=n_itr, env=env),
                            flat_param=torch.arange(4.0)), d / "learner.pt")
    for r in range(world):
        snapshot.save_file(dict(format=FORMAT, itr=itr if shard_itr is None else shard_itr, rank=r, world=world, model=env,
                                precision=precision, state_r=torch.zeros(2, 3)), d / f"rank_{r}.pt")
    snapshot.update_latest(root, itr, world)
    return root


def _tree(path):
    """Every file under `path` with its size and modification time."""
    return {str(p.relative_to(path)): (p.stat().st_size, p.stat().st_mtime_ns) for p in sorted(path.rglob("*"))}


def test_latest_pointer_names_the_last_complete_snapshot_and_older_ones_are_pruned(tmp_path):
    root = _fake(tmp_path, itr=0)
    assert json.loads((root / "latest.json").read_text()) == dict(format=FORMAT, itr=0, world=1, dir="itr_0")
    _fake(tmp_path, itr=100)
    # the pointer moved before the older snapshot went away: a stop between the two leaves two complete snapshots
    assert json.loads((root / "latest.json").read_text())["itr"] == 100 and (root / "itr_0").is_dir()
    # a directory a stopped run had begun after its last complete snapshot is removed as well
    (root / "itr_200").mkdir()
    (root / "itr_200" / "rank_0.pt.tmp").write_bytes(b"partial")
    assert snapshot.prune(root, 100) == ["itr_0", "itr_200"]
    assert sorted(p.name for p in root.iterdir()) == ["itr_100", "latest.json"]
    assert sorted(p.name for p in (root / "itr_100").iterdir()) == ["learner.pt", "rank_0.pt"]   # no *.tmp left behind
    latest, learner, shard = snapshot.load(tmp_path, 0, 1, dict(env="jvrc_walk", precision=64, num_procs=64))
    assert latest["itr"] == learner["itr"] == shard["itr"] == 100 and torch.equal(learner["flat_param"], torch.arange(4.0))


def test_a_file_is_replaced_atomically(tmp_path):
    p = tmp_path / "x.pt"
    snapshot.save_file(dict(a=1), p)
    snapshot.save_file(dict(a=2), p)
    assert torch.load(p, weights_only=True) == dict(a=2) and [q.name for q in tmp_path.iterdir()] == ["x.pt"]


def test_plain_args_keep_plain_values_only(tmp_path):
    ns = argparse.Namespace(env="h1", logdir=tmp_path, n_itr=5, lr=3e-4, seed=None, learn_std=True, fn=print)
    assert snapshot.plain_args(ns) == dict(env="h1", logdir=str(tmp_path), n_itr=5, lr=3e-4, seed=None, learn_std=True)


@pytest.mark.parametrize("case,kw,load_kw,match", [
    ("mixed", dict(itr=4, shard_itr=2), {}, "mixed snapshot: the rank-0 shard file holds iteration 2, latest.json names iteration 4"),
    ("world", dict(world=1), dict(world=2), "world size mismatch"),
    ("num_procs", dict(num_procs=64), dict(expect=dict(num_procs=128)), "num_procs mismatch"),
    ("env", dict(env="jvrc_walk"), dict(expect=dict(env="h1")), "env mismatch"),
    ("precision", dict(precision=64), dict(expect=dict(precision=32)), "precision mismatch"),
])
def test_loader_refuses_a_snapshot_this_run_cannot_continue(tmp_path, case, kw, load_kw, match):
    _fake(tmp_path, **kw)
    before = _tree(tmp_path)
    with pytest.raises(SnapshotError, match=match):
        snapshot.load(tmp_path, 0, load_kw.get("world", 1), load_kw.get("expect"))
    assert _tree(tmp_path) == before


def test_loader_refuses_a_missing_or_foreign_snapshot(tmp_path):
    with pytest.raises(SnapshotError, match="no snapshot"):
        snapshot.load(tmp_path, 0, 1)
    root = _fake(tmp_path, world=2)
    (root / "itr_3" / "rank_1.pt").unlink()
    with pytest.raises(SnapshotError, match="rank-1 shard file .* is missing"):
        snapshot.load(tmp_path, 1, 2)
    (root / "latest.json").write_text(json.dumps(dict(format=FORMAT + 1, itr=3, world=2, dir="itr_3")))
    with pytest.raises(SnapshotError, match="format"):
        snapshot.load(tmp_path, 0, 2)


def _run_dir(tmp_path, num_procs=64, n_itr=10):
    run = tmp_path / "run"
    run.mkdir()
    args = argparse.Namespace(env="jvrc_walk", precision=64, num_procs=num_procs, n_itr=n_itr, yaml=None, seed=0, logdir=run)
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    return run


@pytest.mark.parametrize("case", ["missing", "mixed", "world", "num_procs"])
def test_resume_refuses_before_it_writes_anything(tmp_path, monkeypatch, case):
    import run_experiment as rx
    run = _run_dir(tmp_path, num_procs=128 if case == "num_procs" else 64)
    if case != "missing":
        _fake(run, itr=3, shard_itr=1 if case == "mixed" else None)
    if case == "world":
        monkeypatch.setenv("WORLD_SIZE", "2")
    before = _tree(tmp_path)
    match = dict(missing="no snapshot", mixed="mixed snapshot", world="world size mismatch", num_procs="num_procs mismatch")[case]
    with pytest.raises(SystemExit, match=match):
        rx.main(["resume", "--path", str(run), "--n-itr", "20"])
    assert _tree(tmp_path) == before


def test_resume_of_a_finished_run_has_nothing_to_do(tmp_path, capsys):
    import run_experiment as rx
    run = _run_dir(tmp_path, n_itr=10)
    _fake(run, itr=9, n_itr=10)
    before = _tree(tmp_path)
    assert rx.main(["resume", "--path", str(run)]) is None              # the run's own --n-itr
    assert rx.main(["resume", "--path", str(run), "--n-itr", "10"]) is None
    assert capsys.readouterr().out.count("Nothing to do") == 2
    assert _tree(tmp_path) == before
