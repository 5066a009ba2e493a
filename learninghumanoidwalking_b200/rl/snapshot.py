"""Training snapshots: the whole state of a run at the end of iteration k, so that `run_experiment.py resume` continues it
bit for bit (the reference can only `--continued` from the weights).

Layout under the run directory:

    snapshot/itr_<k>/learner.pt     written once, by rank 0 (the replicas are identical)
    snapshot/itr_<k>/rank_<r>.pt    one shard per rank: its environments' HBM records and its sampler's state
    snapshot/latest.json            {"format", "itr", "world", "dir"}: the last complete snapshot

Every file is written as `<name>.tmp`, flushed to disk and renamed.  After all ranks have written theirs (a barrier), rank 0
replaces latest.json and removes every other `itr_*` directory.  A run stopped at any moment therefore leaves latest.json
naming a complete snapshot.  Every file carries k; a loader that finds files of different iterations refuses to load.

The learner holds the flat parameter buffer (actor then critic; `stds` under --learn-std), both Adam moments, the host step
counts of both optimisers and the device-side Adam step number, observation normalisation, best evaluation, sample count and
elapsed training time.  A shard holds `state_r` / `state_i` (an environment's next control step depends only on this record,
its action, (seed, env id) and the model constants), the worker's current observations, its CUDA noise generator and sample
count, the env's `_fresh` flag, and the CPU torch generator (the minibatch permutation draws from it when no seed is given,
and every rank draws its own).
"""
from __future__ import annotations

import json
import os
import shutil
from pathlib import Path

import torch

FORMAT = 1
LATEST = "latest.json"


class SnapshotError(ValueError):
    """A snapshot that is missing, incomplete, of another format or of another run geometry."""


def snapshot_root(run_dir) -> Path:
    return Path(run_dir) / "snapshot"


def plain_args(args) -> dict:
    """The run's arguments as a dict of plain values (Paths as strings), loadable with torch.load(weights_only=True)."""
    out = {}
    for k, v in sorted(vars(args).items()):
        if isinstance(v, Path):
            v = str(v)
        if v is None or isinstance(v, (bool, int, float, str)):
            out[k] = v
    return out


def _replace_atomic(path: Path, write) -> None:
    tmp = path.with_name(path.name + ".tmp")
    with open(tmp, "wb") as f:
        write(f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def save_file(obj: dict, path: Path) -> None:
    _replace_atomic(Path(path), lambda f: torch.save(obj, f))


def update_latest(root, itr: int, world: int) -> None:
    """Point latest.json at snapshot/itr_<itr> (one atomic rename)."""
    root = Path(root)
    doc = json.dumps(dict(format=FORMAT, itr=int(itr), world=int(world), dir=f"itr_{int(itr)}")).encode()
    _replace_atomic(root / LATEST, lambda f: f.write(doc))


def prune(root, keep_itr: int) -> list:
    """Remove every snapshot/itr_* directory except itr_<keep_itr>: the older ones, and any a stopped run had begun after
    its last complete snapshot.  Returns the names removed."""
    keep = f"itr_{int(keep_itr)}"
    gone = []
    for d in sorted(Path(root).glob("itr_*")):
        if d.is_dir() and d.name != keep:
            shutil.rmtree(d, ignore_errors=True)
            gone.append(d.name)
    return gone


def read_latest(run_dir) -> dict:
    root = snapshot_root(run_dir)
    try:
        latest = json.loads((root / LATEST).read_text())
    except FileNotFoundError:
        raise SnapshotError(f"no snapshot in {run_dir}: {root / LATEST} does not exist (was the run trained with --snapshot?)")
    except (OSError, ValueError) as e:
        raise SnapshotError(f"cannot read {root / LATEST}: {e}")
    if latest.get("format") != FORMAT:
        raise SnapshotError(f"snapshot format {latest.get('format')} in {root / LATEST}, this build reads format {FORMAT}")
    return latest


def _read(path: Path, what: str) -> dict:
    try:
        return torch.load(path, map_location="cpu", weights_only=True)
    except FileNotFoundError:
        raise SnapshotError(f"incomplete snapshot: the {what} file {path} is missing")


def load(run_dir, rank: int, world: int, expect: dict | None = None) -> tuple[dict, dict, dict]:
    """(latest, learner, this rank's shard) of the last complete snapshot of `run_dir`, validated: every file of the same
    iteration as latest.json and of this format, the same world size, and the run geometry in `expect` (any of env,
    precision, num_procs) equal to the snapshot's.  Raises SnapshotError naming the mismatch; reads only."""
    latest = read_latest(run_dir)
    k = latest["itr"]
    if latest.get("world") != world:
        raise SnapshotError(f"world size mismatch: the snapshot was written by {latest.get('world')} rank(s), this run has {world} "
                            "(resuming onto a different number of GPUs is not supported)")
    d = snapshot_root(run_dir) / latest["dir"]
    learner = _read(d / "learner.pt", "learner")
    shard = _read(d / f"rank_{rank}.pt", f"rank-{rank} shard")
    for what, doc in (("learner", learner), (f"rank-{rank} shard", shard)):
        if doc.get("format") != FORMAT:
            raise SnapshotError(f"format mismatch: the {what} file is format {doc.get('format')}, this build reads {FORMAT}")
        if doc.get("itr") != k:
            raise SnapshotError(f"mixed snapshot: the {what} file holds iteration {doc.get('itr')}, latest.json names iteration {k}")
        if doc.get("world") != world:
            raise SnapshotError(f"world size mismatch: the {what} file was written at world {doc.get('world')}, this run has {world}")
    if shard.get("rank") != rank:
        raise SnapshotError(f"the rank-{rank} shard file holds rank {shard.get('rank')}")
    have = dict(env=shard.get("model"), precision=shard.get("precision"), num_procs=learner["args"].get("num_procs"))
    for key, want in (expect or {}).items():
        if have[key] != want:
            raise SnapshotError(f"{key} mismatch: the snapshot has {key}={have[key]!r}, this run has {key}={want!r}")
    return latest, learner, shard


def write(ppo, itr: int, elapsed: float) -> Path:
    """Write the snapshot of `ppo` at the end of iteration `itr` (after its evaluation batches).  Every rank calls this."""
    import torch.distributed as dist
    root = snapshot_root(ppo.save_path)
    d = root / f"itr_{int(itr)}"
    d.mkdir(parents=True, exist_ok=True)
    save_file(ppo.snapshot_shard(itr), d / f"rank_{ppo.rank}.pt")
    if ppo.rank == 0:
        save_file(ppo.snapshot_learner(itr, elapsed), d / "learner.pt")
    if ppo.world > 1:
        dist.barrier()
    if ppo.rank == 0:
        update_latest(root, itr, ppo.world)
        prune(root, itr)
    return d
