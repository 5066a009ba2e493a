#!/usr/bin/env python3
"""run_experiment.py — the reference's entry point (run_experiment.py:105-330) on the H100 path.

    python run_experiment.py train --env jvrc_walk --logdir /tmp/logs --num-procs 4096 --n-itr 100 --seed 0
    python -m torch.distributed.run --nproc-per-node 8 run_experiment.py train --env jvrc_step --num-procs 8192 ...
    python run_experiment.py eval --logdir /tmp/logs [--ep-len 10]
    python run_experiment.py eval --path RUN_DIR --num-envs 4096 [--precision 32] [--report r.json]
    python run_experiment.py train ... --snapshot; python run_experiment.py resume --path RUN_DIR [--n-itr N]

Same sub-commands and flags as the reference.  What differs underneath: `--num-procs` is the number of parallel environment
copies (device resident, sharded by index across the ranks of a torchrun launch) instead of Ray worker processes; there is
no Ray, no MuJoCo and no viewer — `eval` rolls the saved actor out deterministically on one device environment and prints
the per-term reward means; with `--out-dir DIR` it also writes the roll-out as `DIR/<actor file stem>.mp4`, one frame per
control step, ray-cast on the GPU (BatchedHumanoidEnv.render_rgb: inertia boxes, contact geometry, slabs and floor, not
the reference's meshes) and encoded with OpenCV, where the reference's EvaluateEnv uses MuJoCo's offscreen renderer.
Artefacts keep the reference's names and format: `<logdir>/<timestamp>_<env>/experiment.pkl`, `actor_<itr>.pt`,
`critic_<itr>.pt` (whole pickled modules, rl/utils/checkpointer.py:51-83); `train --imitate PATH` also keeps a copy of the
teacher as `teacher.pt` (DESIGN §7.2).  `train --schedule adaptive [--desired-kl 0.01]` adapts the learning rate to the policy's
KL after every minibatch (rsl_rl's schedule, DESIGN §7.3); the rate is printed and logged as `Train/learning_rate`.
`train --push-vel V [--push-interval S]` adds legged_gym-style random pushes to every environment: about every S seconds (default
15) an env's root gets a horizontal velocity change of up to V m/s per axis of its heading frame (DESIGN §7.5).  The periodic
evaluation batches run on the training env and see the pushes too; `resume` rebuilds the env with the run's values, and a run
recorded without them has none.  `eval --num-envs N --push-speeds 0,0.5,1,1.5 [--push-directions 8] [--push-at 2.0]` pushes each
env once, at --push-at seconds, with the speed and direction of its cell of the grid (env i: cell i mod speeds x directions), and
prints the survival of each cell; the batched evaluation never gets the training pushes.  `eval --command forward:0,0.2,0.4
inplace:-0.4,0.4 standing` holds walking commands (DESIGN §7.6): with --num-envs N env i holds the command of cell i mod C and the
run prints the achieved velocities and tracking errors of each cell; without it, the one command is held on the single-env roll-out
(and its video) and re-applied after every reset there.  `eval --footsteps forward:0,0.05,0.1 lateral:left,right backward curved
standing` chooses jvrc_step's stepping-stone plans (DESIGN §7.7): with --num-envs N env i resets with the plan of cell i mod C and the
run prints the falls and footsteps reached of each cell; without it, the one plan is chosen at every reset of the single-env
roll-out (and its video).  `train --env jvrc_step --stair-curriculum H` gives every env a stair level (DESIGN §7.8): its FORWARD
plans climb or descend stairs of 0.01 L m, and L goes up by one after a FORWARD episode that did not fall and reached half its
footsteps, and down by one after one that fell short of half, between 0 and H; the iteration table and TensorBoard show the mean
stair height and the fraction of envs at the top level.
"""
import argparse
import os
import pickle
import platform
import re
import sys
from datetime import datetime
from functools import partial
from pathlib import Path

import torch

_F, _I, _P, _S = float, int, Path, str
# the reference's command line (run_experiment.py:152-260), flag for flag, as data: (flag, argparse keywords)
TRAIN_FLAGS = [
    ("--env", dict(required=True, type=_S)), ("--logdir", dict(default=Path("/tmp/logs"), type=_P, help="run directory root")),
    ("--input-norm-steps", dict(type=_I, default=100000)), ("--n-itr", dict(type=_I, default=20000, help="PPO iterations")),
    ("--lr", dict(type=_F, default=3e-4)), ("--eps", dict(type=_F, default=1e-5, help="Adam epsilon")),
    ("--gamma", dict(type=_F, default=0.99)), ("--lam", dict(type=_F, default=0.95, help="GAE lambda")),
    ("--std-dev", dict(type=_F, default=0.223, help="exploration noise")), ("--learn-std", dict(action="store_true")),
    ("--entropy-coeff", dict(type=_F, default=0.0)), ("--clip", dict(type=_F, default=0.2, help="PPO clip range")),
    ("--minibatch-size", dict(type=_I, default=64)), ("--epochs", dict(type=_I, default=3)),
    ("--num-procs", dict(type=_I, default=4096, help="parallel environment copies over all ranks (the reference: Ray workers)")),
    ("--max-grad-norm", dict(type=_F, default=0.5)), ("--max-traj-len", dict(type=_I, default=400, help="episode horizon")),
    ("--no-mirror", dict(action="store_true", help="train without the SymmetricEnv mirror loss")),
    ("--mirror-coeff", dict(default=0.4, type=_F)), ("--eval-freq", dict(default=100, type=_I, help="checkpoint every N iterations")),
    ("--continued", dict(type=_P, help="actor checkpoint to continue from")), ("--recurrent", dict(action="store_true")),
    ("--imitate", dict(type=_S, default=None)), ("--imitate-coeff", dict(type=_F, default=0.0)),
    ("--yaml", dict(type=_S, default=None)), ("--device", dict(type=_S, default="cuda", choices=["auto", "cuda"])),
    ("--seed", dict(type=_I, default=None)),
    # additions of this build
    ("--precision", dict(type=_I, default=32, choices=[32, 64], help="simulator arithmetic (64 = the reference's float64)")),
    ("--tf32", dict(action="store_true", help="TF32 tensor-core GEMMs in the MLPs (off: fp32 like the reference)")),
    ("--steps-per-env", dict(type=_I, default=None, help="transitions per env per iteration (default: max-traj-len)")),
    ("--minibatch-scale", dict(type=_S, default="auto", choices=["auto", "off"],
                               help="auto: --minibatch-size is scaled by (this rank's batch / 4800) so that an iteration keeps the reference's "
                                    "225 optimiser steps at its default flags; off: --minibatch-size samples per rank, literally")),
    ("--snapshot", dict(action="store_true", help="at every checkpoint, also snapshot the whole training state for `resume`")),
    ("--schedule", dict(type=_S, default="fixed", choices=["fixed", "adaptive"],
                        help="learning rate: fixed at --lr, or adaptive: starts at --lr and follows the minibatch KL (DESIGN §7.3)")),
    ("--desired-kl", dict(type=_F, default=0.01, help="target KL of --schedule adaptive")),
    ("--push-vel", dict(type=_F, default=0.0, help="random root-velocity pushes of up to V m/s per horizontal axis (0: off; DESIGN §7.5)")),
    ("--push-interval", dict(type=_F, default=15.0, help="mean seconds between two random pushes of an env")),
    ("--stair-curriculum", dict(type=_F, default=0.0, help="jvrc_step: a stair level per env up to H m, a multiple of 0.01 in (0, 0.2], "
                                                           "moved by each FORWARD episode (0: off, the reference's schedule; DESIGN §7.8)")),
    ("--action-delay", dict(type=_F, default=0.0, help="random action delays: every reset draws its env's delay uniformly from whole "
                                                       "physics substeps in [0, S] s, S <= control_dt (0: off; DESIGN §7.9)")),
    ("--payload-mass", dict(type=_F, default=0.0, help="random payloads: every reset draws a point mass U(0, M) kg on its env's root "
                                                       "link, M <= half the robot's mass (0: off; DESIGN §7.10)")),
    ("--payload-offset", dict(type=_F, default=0.0, help="with --payload-mass: the payload's offset from the root link's centre of "
                                                         "mass is drawn from U(-R, R)^3 m in the link's frame, R <= 0.25")),
    ("--motor-strength", dict(type=_F, default=0.0, help="random motor strengths: every reset draws each actuated joint's torque scale "
                                                         "from U(1 - R, 1 + R), R in [0, 1] (0: off; DESIGN §7.11)")),
    ("--sensor-noise", dict(type=_F, default=0.0, help="sensor errors: every env observes its robot state with uniform noise of M times "
                                                       "the H1 noise scales, M in [0, 4] (0: off; DESIGN §7.12)")),
    ("--sensor-bias", dict(type=_S, default=None, help="sensor errors: every reset draws its env's IMU roll / pitch offsets from U(-O, O) "
                                                       "rad, gyro offsets from U(-G, G) rad/s and encoder offsets from U(-E, E) rad, "
                                                       "given as O,G,E with O, E <= 0.2 and G <= 0.5 (default: none)")),
]
RESUME_FLAGS = [("--path", dict(type=_P, required=True, help="run directory of a `train --snapshot` run")),
                ("--n-itr", dict(type=_I, default=None, help="PPO iterations in all (default: the run's --n-itr)"))]
EVAL_FLAGS = [("--path", dict(type=_P, default=None)), ("--logdir", dict(type=_P, default=None)),
              ("--out-dir", dict(type=_P, default=None, help="write the roll-out as <out-dir>/<actor file stem>.mp4 "
                                                               "(640x480 at 1/control_dt fps; needs OpenCV, the cv2 module)")),
              ("--ep-len", dict(type=_I, default=10, help="seconds to play")), ("--seed", dict(type=_I, default=None)),
              # batched evaluation (DESIGN §7.4): N environments, one episode each, statistics gathered on the device
              ("--num-envs", dict(type=_I, default=None, help="evaluate on N environments at once, env i = Philox env id i")),
              ("--precision", dict(type=_I, default=None, choices=[32, 64], help="simulator arithmetic of --num-envs (default 64)")),
              ("--report", dict(type=_P, default=None, help="with --num-envs: write the statistics and per-env arrays as JSON")),
              # push-recovery sweep of the batched evaluation (DESIGN §7.5)
              ("--push-speeds", dict(type=_S, default=None, help="with --num-envs: comma-separated push speeds in m/s, e.g. 0,0.5,1,1.5")),
              ("--push-directions", dict(type=_I, default=None, help="push directions, evenly spaced from forward (default 8)")),
              ("--push-at", dict(type=_F, default=None, help="seconds into the episode of the one push (default 2.0)")),
              # held walking commands (DESIGN §7.6)
              ("--command", dict(type=_S, nargs="+", action="extend", default=None,
                                 help="held walking commands MODE[:v1,v2,...]: forward:V m/s, inplace:W rad/s, standing; with "
                                      "--num-envs one cell per (mode, value), else exactly one")),
              # chosen stepping-stone plans of jvrc_step (DESIGN §7.7)
              ("--footsteps", dict(type=_S, nargs="+", action="extend", default=None,
                                   help="jvrc_step footstep plans TYPE[:v1,v2,...]: forward:H (signed stair height, m), "
                                        "lateral:left,right, curved[:plan index,...], backward, standing; with --num-envs one cell "
                                        "per (type, value), else exactly one")),
              # the latency sweep (DESIGN §7.9)
              ("--action-delays", dict(type=_S, default=None,
                                       help="comma-separated action delays in s, whole physics substeps up to control_dt, e.g. "
                                            "0,0.005,0.01,0.02,0.025; with --num-envs one cell per delay, else exactly one")),
              # the payload sweep (DESIGN §7.10)
              ("--payloads", dict(type=_S, default=None,
                                  help="comma-separated payload masses in kg on the root link, at most half the robot's mass, e.g. "
                                       "0,5,10,15,20; with --num-envs one cell per mass, else exactly one")),
              ("--payload-at", dict(type=_S, default=None,
                                    help="with --payloads: the payload's point x,y,z in m in the root link's frame, relative to its "
                                         "centre of mass, each within 0.25 (default 0,0,0)")),
              # the motor-strength sweep (DESIGN §7.11)
              ("--motor-strengths", dict(type=_S, default=None,
                                         help="comma-separated motor strength factors in [0, 2], e.g. 0,0.5,0.8,1,1.2; with --num-envs "
                                              "one cell per factor, else exactly one")),
              ("--motor-joints", dict(type=_S, default=None,
                                      help="with --motor-strengths: comma-separated joint names (get_motor_names()) that get the factor, "
                                           "e.g. R_KNEE,L_KNEE; the others keep 1 (default: every joint)")),
              # the sensor sweep (DESIGN §7.12)
              ("--sensor-errors", dict(type=_S, nargs="+", action="extend", default=None,
                                       help="sensor errors KIND:v1,v2,...: roll:RAD and pitch:RAD (IMU offsets, |v| <= 0.2), "
                                            "encoder:RAD (every motor-position offset, |v| <= 0.2), noise:M (the noise multiplier in "
                                            "[0, 4]); each value is one cell, the rest of the cell 0; with --num-envs one cell per "
                                            "value, else exactly one"))]
ENVS = ("jvrc_walk", "jvrc_step", "h1", "jvrc_walk_terrain", "h1_walk")   # jvrc_walk_terrain is an extension (BASELINE configs[4])
from learninghumanoidwalking_b200.rl.imitation import TEACHER_FILE  # noqa: E402  the copy of `--imitate` that `resume` uses


def print_system_info(args, training=True):
    print("=" * 60)
    print("System Information")
    print("=" * 60)
    print(f"PyTorch version: {torch.__version__}")
    print(f"Platform: {platform.system()} {platform.release()}")
    print(f"CUDA devices: {torch.cuda.device_count()}"
          + (f" ({torch.cuda.get_device_name(0)})" if torch.cuda.is_available() else ""))
    if training:
        print("-" * 60)
        print("Training Configuration")
        print("-" * 60)
        for k, v in (("Environment", args.env), ("Log directory", args.logdir), ("Parallel envs", args.num_procs),
                     ("Learning rate", args.lr), ("Max trajectory length", args.max_traj_len), ("Iterations", args.n_itr),
                     ("Seed", args.seed)):
            print(f"{k}: {v}")
        push_vel = getattr(args, "push_vel", 0.0)
        print(f"Random pushes: up to {push_vel} m/s about every {getattr(args, 'push_interval', 15.0)} s" if push_vel > 0
              else "Random pushes: off")
        stairs = getattr(args, "stair_curriculum", 0.0)
        if stairs:
            print(f"Stair curriculum: levels of 0.01 m up to {stairs} m")
        delay = getattr(args, "action_delay", 0.0)
        print(f"Action delays: up to {delay * 1000:g} ms, drawn at every reset" if delay > 0 else "Action delays: off")
        payload = getattr(args, "payload_mass", 0.0)
        if payload:
            print(f"Payloads: up to {payload:g} kg, offset up to {getattr(args, 'payload_offset', 0.0):g} m per axis, drawn at every reset")
        motor = getattr(args, "motor_strength", 0.0)
        if motor:
            print(f"Motor strengths: U({1 - motor:g}, {1 + motor:g}) per joint, drawn at every reset")
        noise, bias = getattr(args, "sensor_noise", 0.0), _sensor_bias(args)
        if noise or any(bias):
            print(f"Sensor errors: noise x{noise:g}; offsets up to {bias[0]:g} rad roll / pitch, {bias[1]:g} rad/s gyro, {bias[2]:g} rad "
                  "encoders, drawn at every reset")
    print("=" * 60)


def _sensor_bias(args):
    """The run's --sensor-bias as (O, G, E): check_sensor_flags leaves it a tuple; a run without the flag has none."""
    bias = getattr(args, "sensor_bias", None)
    return (0.0, 0.0, 0.0) if bias is None else tuple(bias)


def get_latest_run_dir(logdir):
    logdir = Path(logdir)
    subdirs = [d for d in logdir.iterdir() if d.is_dir()] if logdir.exists() else []
    return max(subdirs, key=lambda d: d.stat().st_mtime) if subdirs else None


def get_latest_actor(run_dir):
    files = list(Path(run_dir).glob("actor_*.pt"))
    if not files:
        return Path(run_dir) / "actor.pt"
    return max(files, key=lambda f: int(m.group(1)) if (m := re.search(r"actor_(\d+)\.pt$", f.name)) else -1)


def import_env(env_name_str):
    """run_experiment.py:87-101: env name -> factory of a device-resident batch of that environment."""
    if env_name_str not in ENVS:
        raise Exception("Check env name! (this build has: " + ", ".join(ENVS) + ")")
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return partial(BatchedHumanoidEnv, model=env_name_str)


def _dist_setup():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        return dist.get_rank(), world, local
    return 0, 1, 0


def make_env_fn(args, rank, world, local):
    """This rank's shard of the `--num-procs` environments, wrapped in SymmetricEnv unless --no-mirror."""
    from learninghumanoidwalking_b200.rl.dist_utils import env_shard
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    Env = import_env(args.env)
    if args.num_procs % world:
        raise SystemExit(f"--num-procs {args.num_procs} is not a multiple of the {world} ranks: every rank must hold the same number "
                         "of environments (each optimiser step is one gradient exchange on every rank)")
    first, n_local = env_shard(rank, world, args.num_procs)
    seed = args.seed if args.seed is not None else 0
    env_fn = partial(Env, n_local, precision=args.precision, seed=seed, first_env_id=first, device=local,
                     max_traj_len=args.max_traj_len, path_to_yaml=args.yaml, push_vel=getattr(args, "push_vel", 0.0),
                     push_interval=getattr(args, "push_interval", 15.0),   # an experiment.pkl without them: no pushes
                     stair_curriculum=getattr(args, "stair_curriculum", 0.0),   # nor a stair curriculum
                     action_delay=getattr(args, "action_delay", 0.0),   # nor action delays
                     payload_mass=getattr(args, "payload_mass", 0.0),   # nor payloads
                     payload_offset=getattr(args, "payload_offset", 0.0),
                     motor_strength=getattr(args, "motor_strength", 0.0),   # nor motor strengths
                     sensor_noise=getattr(args, "sensor_noise", 0.0), sensor_bias=_sensor_bias(args))   # nor sensor errors
    _env = env_fn()
    if not args.no_mirror:
        try:
            r = _env.robot
            env_fn = partial(SymmetricEnv, env_fn, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts,
                             clock_inds=r.clock_inds)
            if rank == 0:
                print("Wrapping in SymmetricEnv.")
        except AttributeError as e:
            print("Warning! Cannot use SymmetricEnv.", e)
    _env.close()
    return env_fn


def check_schedule(args):
    """Refuse a learning-rate schedule this launch cannot run, before any environment or run directory exists."""
    from learninghumanoidwalking_b200.rl import schedule
    kind, desired_kl = schedule.schedule_of(args)
    try:
        schedule.check(kind, desired_kl)
    except ValueError as e:
        raise SystemExit(f"train --schedule {kind}: {e}")
    if kind == "adaptive" and os.environ.get("LHW_FUSED_EXCHANGE", "1") == "0":
        raise SystemExit("train --schedule adaptive: the rate lives on the fused exchange, and LHW_FUSED_EXCHANGE=0 selects the "
                         "baseline exchange, which has no adaptive schedule")


def check_push(args):
    """Refuse random-push flags the env would refuse, before any environment or run directory exists."""
    from learninghumanoidwalking_b200.envs.batched_env import push_interval_steps
    from learninghumanoidwalking_b200.model import load_model
    push_vel, push_interval = getattr(args, "push_vel", 0.0), getattr(args, "push_interval", 15.0)
    import_env(args.env)
    mj = load_model(args.env)
    if args.yaml is not None:
        from learninghumanoidwalking_b200.envs.config import apply_config, load_yaml
        mj = apply_config(mj, load_yaml(args.yaml))
    try:
        push_interval_steps(push_vel, push_interval, mj["cfg"]["control_dt"])
    except ValueError as e:
        raise SystemExit(f"train --push-vel {push_vel} --push-interval {push_interval}: {e}")


def check_stairs(args):
    """Refuse a stair curriculum the env would refuse, before any environment or run directory exists."""
    from learninghumanoidwalking_b200.envs.batched_env import stair_levels
    stairs = getattr(args, "stair_curriculum", 0.0)
    import_env(args.env)
    try:
        stair_levels(args.env, stairs)
    except ValueError as e:
        raise SystemExit(f"train --stair-curriculum {stairs}: {e}")


def check_action_delay(args):
    """Refuse a largest action delay the env would refuse (checked against the model after --yaml), before any environment or
    run directory exists."""
    from learninghumanoidwalking_b200.envs.batched_env import action_delay_substeps
    delay = getattr(args, "action_delay", 0.0)
    cfg = _run_cfg(args.env, args.yaml)
    try:
        action_delay_substeps(delay, cfg["sim_dt"], cfg["control_dt"])
    except ValueError as e:
        raise SystemExit(f"train --action-delay {delay}: {e}")


def check_payload_mass(args):
    """Refuse random payload ranges the env would refuse (the mass against the model after --yaml), before any environment or run
    directory exists."""
    from learninghumanoidwalking_b200.envs.batched_env import check_payload_range
    mass, offset = getattr(args, "payload_mass", 0.0), getattr(args, "payload_offset", 0.0)
    try:
        check_payload_range(mass, offset, _run_model(args.env, args.yaml)["total_mass"])
    except ValueError as e:
        raise SystemExit(f"train --payload-mass {mass} --payload-offset {offset}: {e}")


def check_motor_strength_flag(args):
    """Refuse a random motor-strength range the env would refuse, before any environment or run directory exists."""
    from learninghumanoidwalking_b200.envs.batched_env import check_motor_strength_range
    r = getattr(args, "motor_strength", 0.0)
    try:
        check_motor_strength_range(r)
    except ValueError as e:
        raise SystemExit(f"train --motor-strength {r}: {e}")


def check_sensor_flags(args):
    """Refuse random sensor errors the env would refuse, before any environment or run directory exists; --sensor-bias O,G,E
    becomes the tuple (O, G, E) that experiment.pkl keeps."""
    from learninghumanoidwalking_b200.envs.batched_env import check_sensor_range
    noise, bias = getattr(args, "sensor_noise", 0.0), getattr(args, "sensor_bias", None)
    if isinstance(bias, str):
        try:
            bias = tuple(float(v) for v in bias.split(","))
        except ValueError:
            raise SystemExit(f"train --sensor-bias {bias!r}: expected O,G,E, three comma-separated numbers, e.g. 0.05,0.1,0.02")
    try:
        _, bias = check_sensor_range(noise, (0.0, 0.0, 0.0) if bias is None else bias)
    except ValueError as e:
        raise SystemExit(f"train --sensor-noise {noise} --sensor-bias {getattr(args, 'sensor_bias', None)}: {e}")
    args.sensor_bias = bias


def _run_cfg(env_name, yaml):
    """The model's cfg block after the user's YAML, as the env applies it."""
    return _run_model(env_name, yaml)["cfg"]


def _run_model(env_name, yaml):
    """The model after the user's YAML, as the env applies it."""
    from learninghumanoidwalking_b200.model import load_model
    import_env(env_name)
    mj = load_model(env_name)
    if yaml is not None:
        from learninghumanoidwalking_b200.envs.config import apply_config, load_yaml
        mj = apply_config(mj, load_yaml(yaml))
    return mj


def run_experiment(args):
    from learninghumanoidwalking_b200.rl import PPO
    check_push(args)
    check_stairs(args)
    check_action_delay(args)
    check_payload_mass(args)
    check_motor_strength_flag(args)
    check_sensor_flags(args)
    rank, world, local = _dist_setup()
    timestamp = datetime.now().strftime("%y-%m-%d-%H-%M-%S-%f")[:-3]
    args.logdir = Path(args.logdir) / f"{timestamp}_{args.env}"
    if world > 1 and args.snapshot:
        # every rank writes its shard of a snapshot into the run directory: rank 0's timestamp names it on all of them
        import torch.distributed as dist
        name = [args.logdir]
        dist.broadcast_object_list(name, src=0)
        args.logdir = name[0]
    if rank == 0:
        print_system_info(args)
    if args.recurrent:
        raise NotImplementedError("--recurrent is outside the accelerated path (SURVEY.md §2)")
    check_schedule(args)
    if args.imitate:
        # the teacher, its env and the projector to this env are checked before any environment or run directory exists
        from learninghumanoidwalking_b200.rl import imitation
        import_env(args.env)
        try:
            _, args.imitate_env, _ = imitation.check_teacher(args.imitate, args.env)
        except ValueError as e:
            raise SystemExit(f"train --imitate {args.imitate} for a {args.env} student: {e}")
    env_fn = make_env_fn(args, rank, world, local)
    if rank == 0:
        import shutil
        Path.mkdir(args.logdir, parents=True, exist_ok=True)
        with open(Path(args.logdir, "experiment.pkl"), "wb") as f:
            pickle.dump(args, f)
        if args.yaml is not None:      # run_experiment.py:141-144: the YAML rides along with the run
            shutil.copyfile(args.yaml, Path(args.logdir, Path(args.yaml).name))
        if args.imitate:               # so does the teacher (not actor*.pt: `eval` and get_latest_actor glob that)
            shutil.copyfile(args.imitate, Path(args.logdir, TEACHER_FILE))
    algo = PPO(env_fn, args, seed=args.seed)
    if args.continued is not None:
        actor = torch.load(args.continued, weights_only=False)
        critic = torch.load(Path(args.continued.parent, "critic" + str(args.continued).split("actor")[1]), weights_only=False)
        algo.load_pretrained(actor, critic)
        if rank == 0:
            print("Loaded (pre-trained) actor from: ", args.continued)
    algo.train(env_fn, args.n_itr, verbose=rank == 0)


def resume(args):
    """Continue the run in --path from its last snapshot (`train --snapshot`): the same run, bit for bit, as if it had never
    stopped, up to --n-itr iterations in all (default: the run's own).  Checkpoints, TensorBoard events and snapshots go on
    being written into the same directory.  Launch it with the same number of ranks as the run."""
    from learninghumanoidwalking_b200.rl import PPO, snapshot
    run_dir = Path(args.path)
    try:
        with open(run_dir / "experiment.pkl", "rb") as f:
            run_args = pickle.load(f)
    except FileNotFoundError:
        raise SystemExit(f"resume: {run_dir} is not a run directory (no experiment.pkl)")
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    try:    # refuse a snapshot this launch cannot continue before anything starts or is written
        _, learner, _ = snapshot.load(run_dir, rank, world, dict(env=run_args.env, precision=run_args.precision,
                                                                 num_procs=run_args.num_procs))
    except snapshot.SnapshotError as e:
        raise SystemExit(f"resume: {e}")
    n_itr = args.n_itr if args.n_itr is not None else learner["args"]["n_itr"]
    start = learner["itr"] + 1
    if start >= n_itr:
        if rank == 0:
            print(f"Nothing to do: the snapshot of {run_dir} is at iteration {start - 1} of {n_itr}.")
        return None
    check_schedule(run_args)      # an experiment.pkl without a schedule is a fixed-rate run
    rank, world, local = _dist_setup()
    run_args.logdir, run_args.n_itr, run_args.snapshot = run_dir, n_itr, True
    if run_args.yaml is not None and Path(run_dir, Path(run_args.yaml).name).exists():
        run_args.yaml = str(Path(run_dir, Path(run_args.yaml).name))     # the copy that rode along with the run
    if getattr(run_args, "imitate", None) and Path(run_dir, TEACHER_FILE).exists():
        run_args.imitate = str(Path(run_dir, TEACHER_FILE))              # its env is run_args.imitate_env
    if rank == 0:
        print_system_info(run_args)
        print(f"Resuming {run_dir} after iteration {start - 1}.")
    env_fn = make_env_fn(run_args, rank, world, local)
    algo = PPO(env_fn, run_args, seed=run_args.seed)
    algo.restore(run_dir)
    return algo.train(env_fn, n_itr, verbose=rank == 0, start_itr=start)


def find_actor(args):
    """The actor file `eval --path / --logdir` names."""
    if args.path is not None:
        if args.path.is_file() and args.path.suffix == ".pt":
            path_to_actor = args.path
        elif args.path.is_dir():
            path_to_actor = get_latest_actor(args.path)
        else:
            raise Exception("Invalid path to actor module: ", args.path)
    elif args.logdir is not None:
        latest = get_latest_run_dir(args.logdir)
        if latest is None:
            raise Exception(f"No run directories found under: {args.logdir}")
        path_to_actor = get_latest_actor(latest)
    else:
        raise Exception("Must provide either --path or --logdir")
    return path_to_actor


def push_sweep(args):
    """The push-recovery grid of `eval --num-envs N --push-speeds ...` as dict(speeds, directions, push_at), or None without push
    flags; refuses a grid that cannot be run before anything is loaded."""
    if args.push_speeds is None:
        if args.push_directions is not None or args.push_at is not None:
            raise SystemExit("eval --push-directions and --push-at describe the push sweep: add --push-speeds")
        return None
    try:
        speeds = [float(v) for v in args.push_speeds.split(",")]
    except ValueError:
        raise SystemExit(f"eval --push-speeds {args.push_speeds!r}: expected comma-separated speeds in m/s, e.g. 0,0.5,1,1.5")
    if not all(v >= 0 and v < float("inf") for v in speeds):
        raise SystemExit(f"eval --push-speeds {args.push_speeds}: every speed must be finite and >= 0")
    directions = 8 if args.push_directions is None else args.push_directions
    if directions < 1:
        raise SystemExit(f"eval --push-directions {directions}: needs at least one direction")
    cells = len(speeds) * directions
    if args.num_envs < cells:
        raise SystemExit(f"eval --num-envs {args.num_envs}: the push grid has {len(speeds)} speeds x {directions} directions = {cells} "
                         "cells, and every cell needs at least one environment")
    push_at = 2.0 if args.push_at is None else args.push_at
    if not push_at < float("inf"):
        raise SystemExit(f"eval --push-at {push_at}: must be a finite number of seconds")
    return dict(speeds=speeds, directions=directions, push_at=push_at)


COMMAND_MODES = {"forward": "FORWARD", "inplace": "INPLACE", "standing": "STANDING"}


def command_cells(args):
    """The held commands of `eval --command ...` as [(mode name, value), ...] (rl/evaluation.py MODES), or None without the flag;
    refuses a list that cannot be run before anything is loaded.  Values outside the training ranges are allowed."""
    if args.command is None:
        return None
    cells = []
    for spec in args.command:
        name, sep, values = spec.partition(":")
        if name not in COMMAND_MODES:
            raise SystemExit(f"eval --command {spec!r}: unknown mode {name!r}; expected forward:V[,V...], inplace:W[,W...] or standing")
        if name == "standing":
            if sep:
                raise SystemExit(f"eval --command {spec!r}: standing takes no values")
            cells.append(("STANDING", 0.0))
            continue
        try:
            vs = [float(v) for v in values.split(",")]
        except ValueError:
            raise SystemExit(f"eval --command {spec!r}: expected {name}:V[,V...] with comma-separated numbers "
                             f"({'m/s' if name == 'forward' else 'rad/s'})")
        if not all(abs(v) < float("inf") for v in vs):
            raise SystemExit(f"eval --command {spec!r}: every value must be finite")
        cells += [(COMMAND_MODES[name], v) for v in vs]
    if args.push_speeds is not None:
        raise SystemExit("eval --command and --push-speeds are separate sweeps: run them one at a time")
    if args.num_envs is None and len(cells) > 1:
        raise SystemExit(f"eval --command: {len(cells)} commands need the batched evaluation (add --num-envs N); the single-env "
                         "roll-out holds exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --command lists {len(cells)} cells, and every cell needs at least one "
                         "environment")
    return cells


def check_command_env(env_name):
    """Refuse --command for a run whose env has no walking command, before its actor is loaded."""
    from learninghumanoidwalking_b200.envs.batched_env import COMMAND_ENVS
    if env_name not in COMMAND_ENVS:
        raise SystemExit(f"eval --command: the run's env {env_name} has no walking command; only {', '.join(COMMAND_ENVS)} take one")


def footstep_cells(args):
    """The chosen plans of `eval --footsteps ...` as [(plan type name, value), ...] (envs/batched_env.py FOOTSTEP_MODES), or None
    without the flag; refuses a list that cannot be run before anything is loaded.  Bare `curved` is a curved plan drawn at the
    reset (value -1)."""
    if args.footsteps is None:
        return None
    from learninghumanoidwalking_b200.model import load_model
    st = load_model("jvrc_step")["stepping"]
    nplan, max_h = len(st["plans"]), 2 * float(st["slab_half"][2])
    cells = []
    for spec in args.footsteps:
        name, sep, values = spec.partition(":")
        if name not in ("forward", "lateral", "curved", "backward", "standing"):
            raise SystemExit(f"eval --footsteps {spec!r}: unknown plan type {name!r}; expected forward:H[,H...], lateral:left,right, "
                             "curved[:I,...], backward or standing")
        if name in ("backward", "standing") or (name == "curved" and not sep):
            if sep:
                raise SystemExit(f"eval --footsteps {spec!r}: {name} takes no values")
            cells.append((name.upper(), -1.0 if name == "curved" else 0.0))
            continue
        if name == "lateral":
            sides = values.split(",")
            if not all(v in ("left", "right") for v in sides):
                raise SystemExit(f"eval --footsteps {spec!r}: expected lateral:left, lateral:right or lateral:left,right")
            cells += [("LATERAL", 1.0 if v == "left" else -1.0) for v in sides]
            continue
        try:
            vs = [float(v) for v in values.split(",")]
        except ValueError:
            raise SystemExit(f"eval --footsteps {spec!r}: expected {name}:" +
                             ("H[,H...] with comma-separated stair heights in m" if name == "forward" else "I[,I...] with plan indices"))
        if not all(abs(v) < float("inf") for v in vs):
            raise SystemExit(f"eval --footsteps {spec!r}: every value must be finite")
        if name == "forward" and any(abs(v) > max_h for v in vs):
            raise SystemExit(f"eval --footsteps {spec!r}: a stair height must lie in [-{max_h:g}, {max_h:g}] m (twice a slab's half "
                             "height: above it a slab's side face no longer covers the riser below the next slab)")
        if name == "curved" and any(v != int(v) or not 0 <= v < nplan for v in vs):
            raise SystemExit(f"eval --footsteps {spec!r}: a curved plan index must be an integer in [0, {nplan})")
        cells += [(name.upper(), v) for v in vs]
    if args.push_speeds is not None or args.command is not None:
        raise SystemExit("eval --footsteps, --command and --push-speeds are separate sweeps: run them one at a time")
    if args.num_envs is None and len(cells) > 1:
        raise SystemExit(f"eval --footsteps: {len(cells)} plans need the batched evaluation (add --num-envs N); the single-env "
                         "roll-out takes exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --footsteps lists {len(cells)} cells, and every cell needs at least one "
                         "environment")
    return cells


def delay_cells(args):
    """The action delays of `eval --action-delays ...` in seconds, or None without the flag; the grammar and the combinations are
    refused here, the values against the run's model by check_delays."""
    if args.action_delays is None:
        return None
    try:
        cells = [float(v) for v in args.action_delays.split(",")]
    except ValueError:
        raise SystemExit(f"eval --action-delays {args.action_delays!r}: expected comma-separated delays in s, e.g. 0,0.005,0.01,0.02")
    if not all(v >= 0 and v < float("inf") for v in cells):
        raise SystemExit(f"eval --action-delays {args.action_delays}: every delay must be finite and >= 0")
    if args.push_speeds is not None or args.command is not None or args.footsteps is not None:
        raise SystemExit("eval --action-delays, --push-speeds, --command and --footsteps are separate sweeps: run them one at a time")
    if args.num_envs is None and len(cells) != 1:
        raise SystemExit(f"eval --action-delays: {len(cells)} delays need the batched evaluation (add --num-envs N); the single-env "
                         "roll-out takes exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --action-delays lists {len(cells)} cells, and every cell needs at least "
                         "one environment")
    return cells


def check_delays(delays, run_args, yaml):
    """Refuse delays the run's env would refuse (whole substeps of its sim_dt, at most its control_dt), before the actor is
    loaded."""
    from learninghumanoidwalking_b200.envs.batched_env import action_delay_substeps
    cfg = _run_cfg(run_args.env, yaml)
    try:
        action_delay_substeps(delays, cfg["sim_dt"], cfg["control_dt"])
    except ValueError as e:
        raise SystemExit(f"eval --action-delays: {e}")


def payload_cells(args):
    """The payload masses of `eval --payloads ...` in kg and the one offset of --payload-at, or None without the flag; the
    grammar, the offset and the combinations are refused here, the masses against the run's model by check_payloads."""
    if args.payloads is None:
        if args.payload_at is not None:
            raise SystemExit("eval --payload-at places the payload of --payloads: add --payloads")
        return None
    try:
        cells = [float(v) for v in args.payloads.split(",")]
    except ValueError:
        raise SystemExit(f"eval --payloads {args.payloads!r}: expected comma-separated masses in kg, e.g. 0,5,10,15,20")
    if not all(v >= 0 and v < float("inf") for v in cells):
        raise SystemExit(f"eval --payloads {args.payloads}: every mass must be finite and >= 0")
    try:
        at = [0.0, 0.0, 0.0] if args.payload_at is None else [float(v) for v in args.payload_at.split(",")]
    except ValueError:
        at = []
    if len(at) != 3:
        raise SystemExit(f"eval --payload-at {args.payload_at!r}: expected one point x,y,z in m, e.g. 0,0,0.1")
    from learninghumanoidwalking_b200.envs.batched_env import PAYLOAD_MAX_OFFSET
    if not all(abs(v) <= PAYLOAD_MAX_OFFSET for v in at):
        raise SystemExit(f"eval --payload-at {args.payload_at}: every coordinate must be finite and within {PAYLOAD_MAX_OFFSET:g} m")
    if (args.push_speeds is not None or args.command is not None or args.footsteps is not None
            or args.action_delays is not None):
        raise SystemExit("eval --payloads, --push-speeds, --command, --footsteps and --action-delays are separate sweeps: run them "
                         "one at a time")
    if args.num_envs is None and len(cells) != 1:
        raise SystemExit(f"eval --payloads: {len(cells)} masses need the batched evaluation (add --num-envs N); the single-env "
                         "roll-out takes exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --payloads lists {len(cells)} cells, and every cell needs at least one "
                         "environment")
    return dict(masses=cells, at=at)


def check_payloads(payloads, run_args, yaml):
    """Refuse masses the run's env would refuse (at most half its total_mass), before the actor is loaded."""
    from learninghumanoidwalking_b200.envs.batched_env import check_payload
    try:
        check_payload(payloads["masses"], payloads["at"], _run_model(run_args.env, yaml)["total_mass"])
    except ValueError as e:
        raise SystemExit(f"eval --payloads: {e}")


def motor_cells(args):
    """The strength factors of `eval --motor-strengths ...` and the joint names of --motor-joints (None: every joint), or None
    without the flag; the grammar, the range and the combinations are refused here, the joint names against the run's model by
    motor_joint_mask."""
    if args.motor_strengths is None:
        if args.motor_joints is not None:
            raise SystemExit("eval --motor-joints names the joints of --motor-strengths: add --motor-strengths")
        return None
    try:
        cells = [float(v) for v in args.motor_strengths.split(",")]
    except ValueError:
        raise SystemExit(f"eval --motor-strengths {args.motor_strengths!r}: expected comma-separated factors, e.g. 0,0.5,0.8,1,1.2")
    from learninghumanoidwalking_b200.envs.batched_env import check_motor_strength
    try:
        check_motor_strength(cells)
    except ValueError as e:
        raise SystemExit(f"eval --motor-strengths {args.motor_strengths}: {e}")
    joints = None
    if args.motor_joints is not None:
        joints = [j.strip() for j in args.motor_joints.split(",")]
        if not all(joints):
            raise SystemExit(f"eval --motor-joints {args.motor_joints!r}: expected comma-separated joint names, e.g. R_KNEE,L_KNEE")
    if (args.push_speeds is not None or args.command is not None or args.footsteps is not None
            or args.action_delays is not None or args.payloads is not None):
        raise SystemExit("eval --motor-strengths, --push-speeds, --command, --footsteps, --action-delays and --payloads are separate "
                         "sweeps: run them one at a time")
    if args.num_envs is None and len(cells) != 1:
        raise SystemExit(f"eval --motor-strengths: {len(cells)} factors need the batched evaluation (add --num-envs N); the "
                         "single-env roll-out takes exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --motor-strengths lists {len(cells)} cells, and every cell needs at "
                         "least one environment")
    return dict(factors=cells, joints=joints)


def motor_joint_mask(motor, run_args, yaml):
    """The [NU] bools of the joints --motor-joints names, in the run's model's joint order (every joint without the flag);
    an unknown name is refused before the actor is loaded.  The joint names go into `motor` too."""
    names = [lk["joint"]["name"] for lk in _run_model(run_args.env, yaml)["links"][1:]]
    if motor["joints"] is None:
        motor["joints"] = names
    unknown = [j for j in motor["joints"] if j not in names]
    if unknown:
        raise SystemExit(f"eval --motor-joints: {', '.join(unknown)} is not a joint of the run's {run_args.env} model; its joints are "
                         f"{', '.join(names)}")
    motor["mask"] = [n in motor["joints"] for n in names]
    return motor["mask"]


def sensor_cells(args):
    """The cells of `eval --sensor-errors KIND:v1,v2 ...` as [(kind, value), ...] (rl/evaluation.py SENSOR_KINDS), or None without
    the flag; the grammar, the ranges, the cell count and the combinations are refused here, before anything is loaded."""
    if args.sensor_errors is None:
        return None
    from learninghumanoidwalking_b200.envs.batched_env import SENSOR_MAX_BIAS, SENSOR_MAX_NOISE
    from learninghumanoidwalking_b200.rl.evaluation import SENSOR_KINDS
    cells = []
    for spec in args.sensor_errors:
        kind, _, values = spec.partition(":")
        if kind not in SENSOR_KINDS:
            raise SystemExit(f"eval --sensor-errors {spec!r}: unknown kind {kind!r}; expected roll:V[,V...], pitch:V[,V...], "
                             "encoder:V[,V...] or noise:M[,M...]")
        try:
            vs = [float(v) for v in values.split(",")]
        except ValueError:
            raise SystemExit(f"eval --sensor-errors {spec!r}: expected {kind}:V[,V...] with comma-separated numbers")
        lo, hi = (0.0, SENSOR_MAX_NOISE) if kind == "noise" else (-SENSOR_MAX_BIAS[0 if kind != "encoder" else 2],
                                                                  SENSOR_MAX_BIAS[0 if kind != "encoder" else 2])
        for v in vs:
            if not lo <= v <= hi:
                raise SystemExit(f"eval --sensor-errors {spec!r}: a {kind} value must lie in [{lo:g}, {hi:g}], got {v}")
        cells += [(kind, v) for v in vs]
    if (args.push_speeds is not None or args.command is not None or args.footsteps is not None or args.action_delays is not None
            or args.payloads is not None or args.motor_strengths is not None):
        raise SystemExit("eval --sensor-errors, --push-speeds, --command, --footsteps, --action-delays, --payloads and "
                         "--motor-strengths are separate sweeps: run them one at a time")
    if args.num_envs is None and len(cells) != 1:
        raise SystemExit(f"eval --sensor-errors: {len(cells)} cells need the batched evaluation (add --num-envs N); the single-env "
                         "roll-out takes exactly one")
    if args.num_envs is not None and args.num_envs < len(cells):
        raise SystemExit(f"eval --num-envs {args.num_envs}: --sensor-errors lists {len(cells)} cells, and every cell needs at least "
                         "one environment")
    return cells


def check_footstep_env(env_name):
    """Refuse --footsteps for a run whose env is not jvrc_step, before its actor is loaded."""
    if env_name != "jvrc_step":
        raise SystemExit(f"eval --footsteps: the run's env {env_name} has no footstep plan; only jvrc_step (SteppingTask) takes one")


def evaluate_batched(args):
    """`eval --num-envs N`: the deterministic actor on N environments of the run's env, horizon and YAML, one episode each
    (rl/evaluation.py), with a table of the outcomes and, with --report, the JSON report."""
    if args.num_envs < 1:
        raise SystemExit(f"eval --num-envs {args.num_envs}: needs at least one environment")
    if args.out_dir is not None:
        raise SystemExit("eval --out-dir renders one roll-out to video; it cannot be combined with --num-envs")
    push = push_sweep(args)
    commands = command_cells(args)
    footsteps = footstep_cells(args)
    delays = delay_cells(args)
    payloads = payload_cells(args)
    motor = motor_cells(args)
    sensor = sensor_cells(args)
    path_to_actor = find_actor(args)
    print(f"Loading model: {path_to_actor}")
    with open(Path(path_to_actor.parent, "experiment.pkl"), "rb") as f:
        run_args = pickle.load(f)
    if commands is not None:
        check_command_env(run_args.env)
    if footsteps is not None:
        check_footstep_env(run_args.env)
    yaml = run_args.yaml
    if yaml is not None and Path(path_to_actor.parent, Path(yaml).name).exists():
        yaml = str(Path(path_to_actor.parent, Path(yaml).name))      # the copy that rode along with the run, as `resume` uses
    if delays is not None:
        check_delays(delays, run_args, yaml)
    if payloads is not None:
        check_payloads(payloads, run_args, yaml)
    if motor is not None:
        motor_joint_mask(motor, run_args, yaml)
    if push is not None:       # the push step needs the run's control step and horizon; refused before the actor is loaded
        from learninghumanoidwalking_b200.envs.config import apply_config, load_yaml
        from learninghumanoidwalking_b200.model import load_model
        import_env(run_args.env)
        mj = load_model(run_args.env)
        dt = (apply_config(mj, load_yaml(yaml)) if yaml is not None else mj)["cfg"]["control_dt"]
        k = int(round(push["push_at"] / dt))
        if not 1 <= k < run_args.max_traj_len:
            raise SystemExit(f"eval --push-at {push['push_at']}: the push comes after control step {k} of {dt} s, which must lie in "
                             f"1..{run_args.max_traj_len - 1} (the run's horizon is {run_args.max_traj_len} steps)")
    from learninghumanoidwalking_b200.rl.evaluation import evaluate_batched as run
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    policy = torch.load(path_to_actor, weights_only=False).cuda().eval()
    print_system_info(args, training=False)
    precision = 64 if args.precision is None else args.precision
    env = import_env(run_args.env)(args.num_envs, precision=precision, seed=args.seed or 0,
                                   max_traj_len=run_args.max_traj_len, path_to_yaml=yaml)
    report = run(policy, env, args.report, meta=dict(actor=str(path_to_actor), yaml=yaml), push=push, commands=commands,
                 footsteps=footsteps, delays=delays, payloads=payloads, motor=motor, sensor=sensor)
    env.close()
    return report


def evaluate(args):
    """Deterministic roll-out of a saved actor on one device environment (the numbers EvaluateEnv would overlay)."""
    if args.num_envs is not None:
        return evaluate_batched(args)
    if args.precision is not None or args.report is not None:
        raise SystemExit("eval --precision and --report belong to the batched evaluation: add --num-envs N")
    if args.push_speeds is not None or args.push_directions is not None or args.push_at is not None:
        raise SystemExit("eval --push-speeds, --push-directions and --push-at belong to the batched evaluation: add --num-envs N")
    commands = command_cells(args)
    footsteps = footstep_cells(args)
    delays = delay_cells(args)
    payloads = payload_cells(args)
    motor = motor_cells(args)
    sensor = sensor_cells(args)
    path_to_actor = find_actor(args)
    print(f"Loading model: {path_to_actor}")
    with open(Path(path_to_actor.parent, "experiment.pkl"), "rb") as f:
        run_args = pickle.load(f)
    if commands is not None:
        check_command_env(run_args.env)
    if footsteps is not None:
        check_footstep_env(run_args.env)
    if delays is not None:
        check_delays(delays, run_args, None)     # the single-env roll-out runs the env's own model, as it always has
    if payloads is not None:
        check_payloads(payloads, run_args, None)
    if motor is not None:
        motor_joint_mask(motor, run_args, None)
    cv2 = None
    if args.out_dir is not None:
        try:
            import cv2
        except ImportError as e:
            raise SystemExit(f"eval --out-dir writes the video with OpenCV, and the cv2 module could not be imported ({e}); "
                             "install opencv-python or opencv-python-headless")
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()   # a checkpoint pickles the reference's module names; a fresh `eval` process has not imported them
    policy = torch.load(path_to_actor, weights_only=False).cuda().eval()
    print_system_info(args, training=False)
    env = import_env(run_args.env)(1, precision=64, seed=args.seed or 0)
    if sensor is not None:           # the one cell, set once: explicit errors hold through every reset, the first one included
        from learninghumanoidwalking_b200.rl.evaluation import sensor_grid
        env.set_sensor_errors(*sensor_grid(1, sensor, env.act_dim)[1:])

    def reset():
        if footsteps is not None:     # the one plan, chosen again at every reset
            from learninghumanoidwalking_b200.rl.evaluation import footstep_grid
            env.reset_footsteps(*footstep_grid(1, footsteps))
        else:
            env.reset()
        if commands is not None:     # the one command, held again after every reset
            from learninghumanoidwalking_b200.rl.evaluation import command_grid, command_refs
            mode, value = command_grid(1, commands)
            env.set_command(mode, command_refs(mode, value))
        if delays is not None:       # the one delay, set again after every reset
            env.set_action_delay(delays)
        if payloads is not None:     # the one payload, set again after every reset (the video does not draw it)
            env.set_payload(payloads["masses"], payloads["at"])
        if motor is not None:        # the one strength on the named joints, set again after every reset
            env.set_motor_strength([[motor["factors"][0] if on else 1.0 for on in motor["mask"]]])
        return env.obs.float()

    obs = reset()
    n_steps = int(args.ep_len / env.dt)
    video = None
    if cv2 is not None:
        args.out_dir.mkdir(parents=True, exist_ok=True)
        video_path = args.out_dir / (path_to_actor.stem + ".mp4")
        video = cv2.VideoWriter(str(video_path), cv2.VideoWriter_fourcc(*"mp4v"), 1.0 / env.dt, (640, 480))
        if not video.isOpened():
            raise SystemExit(f"eval --out-dir: OpenCV cannot write {video_path} with the mp4v codec")

    def frame():
        if video is not None:
            video.write(env.render_rgb((0,), 640, 480)[0].flip(-1).cpu().numpy())   # RGB -> OpenCV's BGR

    frame()
    totals, ep_ret, ep_len, episodes = torch.zeros(10, dtype=env.dtype, device=env.device), 0.0, 0, []
    with torch.no_grad():
        for _ in range(n_steps):
            obs, rew, done, _ = env.step(policy(obs, deterministic=True).to(env.dtype), autoreset=False)
            frame()
            totals += env.rew_terms[0]
            ep_ret, ep_len = ep_ret + float(rew[0]), ep_len + 1
            if bool(done[0]):
                episodes.append((ep_len, ep_ret))
                ep_ret, ep_len = 0.0, 0
                obs = reset()
            obs = obs.float()
    episodes.append((ep_len, ep_ret))
    print(f"{len(episodes)} episode(s) in {n_steps} control steps: " + ", ".join(f"len {l} return {r:.2f}" for l, r in episodes))
    for name, v in zip(env.reward_names, (totals / n_steps).tolist()):
        print(f"  mean {name:>20s} {v:.4f}")
    if video is not None:
        video.release()
        print(f"Wrote {video_path} ({n_steps + 1} frames)")
    env.close()
    return episodes


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    parser = argparse.ArgumentParser()
    if argv and argv[0] == "train":
        for flag, kw in TRAIN_FLAGS:
            parser.add_argument(flag, **kw)
        args = parser.parse_args(argv[1:])
        if args.seed is not None:
            torch.manual_seed(args.seed)
            print(f"Deterministic mode enabled with seed: {args.seed}")
        return run_experiment(args)
    elif argv and argv[0] == "eval":
        for flag, kw in EVAL_FLAGS:
            parser.add_argument(flag, **kw)
        args = parser.parse_args(argv[1:])
        return evaluate(args)
    elif argv and argv[0] == "resume":
        for flag, kw in RESUME_FLAGS:
            parser.add_argument(flag, **kw)
        args = parser.parse_args(argv[1:])
        return resume(args)
    else:
        parser.error("usage: run_experiment.py {train,eval,resume} ...")


if __name__ == "__main__":
    main()
