"""Imitation of a saved actor: `train --imitate PATH --imitate-coeff C` (the term of rl/algos/ppo.py:361-368).

The reference's rl/algos/imitation.py is not in this tree, so the teacher's format and the projector are build-defined
(DESIGN §7.2):
  * the teacher is a whole pickled actor (`torch.save(module)`, this build's or the reference's), run as
    `teacher(teacher_obs, deterministic=True)` with its own embedded obs_mean / obs_std;
  * the projector maps a student observation batch [B, S] to the teacher's input [B, T] and an optional per-sample
    mask [B, 1]; it is chosen by the pair (teacher env, student env):
      - the same observation layout (the same env, or jvrc_walk <-> jvrc_walk_terrain): the identity, no mask;
      - an h1 teacher for an h1_walk student: the 35 robot-state words h1_walk's observation starts with, masked to the
        samples whose walking-task mode is STANDING (the one-hot word 39: FORWARD, INPLACE, STANDING at NROBOT+2..+4 of
        csrc/sim_core.h env_obs) -- the standing teacher teaches the standing samples only;
      - any other pair raises ValueError;
  * the teacher's env is `env` of the experiment.pkl next to the teacher file (both the reference and this build write one);
    without it only the identity between equal widths is allowed.
"""
from __future__ import annotations

import pickle
from pathlib import Path

import torch

# observation / action widths of each environment (csrc/sim_core.h Dims; envs/batched_env.py checks them at creation)
ENV_DIMS = {"jvrc_walk": (37, 12), "jvrc_walk_terrain": (37, 12), "jvrc_step": (39, 12), "h1": (35, 10), "h1_walk": (43, 10)}
SAME_LAYOUT = ({"jvrc_walk", "jvrc_walk_terrain"},)
H1_ROBOT_WORDS = 35          # h1_walk = h1's 35 robot-state words, then the 8 walking-task words (DESIGN §4.6)
H1_WALK_STANDING_WORD = 39   # NROBOT + 4: the STANDING word of the mode one-hot
TEACHER_FILE = "teacher.pt"   # the copy of `--imitate` in a run directory (not actor*.pt: `eval` globs that)


class IdentityProjector:
    """The teacher reads the student's observation as it is; every sample counts."""

    def __call__(self, obs):
        return obs, None


class H1StandingProjector:
    """h1 teacher -> h1_walk student: the robot-state words, masked to the STANDING samples."""

    def __call__(self, obs):
        return obs[:, :H1_ROBOT_WORDS], obs[:, H1_WALK_STANDING_WORD:H1_WALK_STANDING_WORD + 1]


def make_projector(teacher_env, student_env, teacher_in, teacher_act, student_obs, student_act):
    """The projector for a teacher of input / action width (teacher_in, teacher_act) trained on `teacher_env` (None: unknown)
    and a student on `student_env` with widths (student_obs, student_act).  Raises ValueError naming both sides."""
    who = f"a {teacher_env or 'teacher of unknown env'} teacher (input {teacher_in}, {teacher_act} actions) and a {student_env} student " \
          f"(observation {student_obs}, {student_act} actions)"
    if teacher_act != student_act:
        raise ValueError(f"imitation: the action widths differ between {who}")
    if teacher_env is None:
        if teacher_in == student_obs:
            return IdentityProjector()
        raise ValueError(f"imitation: no experiment.pkl names the teacher's env, and the identity does not fit {who}")
    same = teacher_env == student_env or any({teacher_env, student_env} == s for s in SAME_LAYOUT)
    if same and teacher_in == student_obs:
        return IdentityProjector()
    if (teacher_env, student_env) == ("h1", "h1_walk") and teacher_in == H1_ROBOT_WORDS and student_obs > H1_WALK_STANDING_WORD:
        return H1StandingProjector()
    raise ValueError(f"imitation: no projector for {who}; supported pairs: the same env, jvrc_walk <-> jvrc_walk_terrain, "
                     "h1 -> h1_walk")


def teacher_env_of(path):
    """The env the teacher file was trained on, or None where nothing says: `env` of the experiment.pkl next to it.  A
    TEACHER_FILE sits in the run directory of a student, whose experiment.pkl records the teacher's env as `imitate_env`."""
    pkl = Path(path).parent / "experiment.pkl"
    if not pkl.is_file():
        return None
    with open(pkl, "rb") as f:
        run = pickle.load(f)
    if Path(path).name == TEACHER_FILE:
        return getattr(run, "imitate_env", None)
    return getattr(run, "env", None)


def load_teacher(path):
    """The pickled actor at `path` on the CPU (the reference's class names resolve to this package's classes); raises
    ValueError naming the file when it is missing or is not an actor."""
    from .policies import install_reference_aliases
    path = Path(path)
    if not path.is_file():
        raise ValueError(f"imitation: the teacher {path} does not exist")
    install_reference_aliases()
    try:
        module = torch.load(path, map_location="cpu", weights_only=False)
    except Exception as e:
        raise ValueError(f"imitation: the teacher {path} does not load: {e}") from e
    if not isinstance(module, torch.nn.Module) or teacher_widths(module) is None:
        raise ValueError(f"imitation: the teacher {path} is not a saved actor (torch.save of a Gaussian_FF_Actor)")
    return module


def teacher_widths(module):
    """(input width, action width) of a saved actor, or None."""
    layers, means = getattr(module, "actor_layers", None), getattr(module, "means", None)
    if layers is None or means is None or not len(layers):
        return None
    return layers[0].in_features, means.out_features


def check_teacher(path, student_env, teacher_env=None):
    """Load the teacher and build its projector for `student_env` without a device or an environment: everything
    `train --imitate` can refuse is refused here, before a run directory exists.  Returns (teacher module, teacher env,
    projector)."""
    module = load_teacher(path)
    if teacher_env is None:
        teacher_env = teacher_env_of(path)
    t_in, t_act = teacher_widths(module)
    s_obs, s_act = ENV_DIMS[student_env]
    try:
        proj = make_projector(teacher_env, student_env, t_in, t_act, s_obs, s_act)
    except ValueError as e:
        raise ValueError(f"{e} (teacher file {path})") from None
    return module, teacher_env, proj


def to_device(module, device):
    """The teacher on `device`, frozen and in eval mode.  The reference's class keeps obs_mean / obs_std / stds as plain
    tensor attributes that .to() does not move, so they are moved by hand (as rl/algos/ppo.py:136-147 does)."""
    module = module.to(device).eval().requires_grad_(False)
    for name in ("obs_mean", "obs_std", "stds"):
        v = module.__dict__.get(name)
        if torch.is_tensor(v):
            module.__dict__[name] = v.to(device, torch.float32)
    return module
