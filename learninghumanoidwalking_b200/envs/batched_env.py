"""BatchedHumanoidEnv — N device-resident copies of a reference humanoid env stepped by one CUDA launch.

Mirrors, per environment, the reference's env protocol (envs/common/base_humanoid_env.py:177-276,
envs/jvrc/jvrc_walk.py): `reset() -> obs`, `step(actions) -> (obs, reward, done, info)`, `observation_space`,
`action_space`, `obs_mean`, `obs_std`, `robot.{mirrored_obs, mirrored_acts, clock_inds, iteration_count}`.
All state lives in two torch CUDA tensors (the HBM records the kernel streams); nothing touches the host
inside a control step.
"""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import numpy as np
import torch

from .. import _lib
from ..model import load_model, pack_model
from ..model.loader import curriculum_height

REWARD_NAMES = ("foot_frc_score", "foot_vel_score", "root_accel", "height_error", "com_vel_error", "yaw_vel_error",
                "upper_body_reward", "posture_error", "torque_penalty", "action_penalty")  # tasks/walking_task.py:131-146
STAND_REWARD_NAMES = ("com_vel_error", "yaw_vel_error", "height", "upperbody", "joint_torque_reward",
                      "posture")                                                          # tasks/standing_task.py:97-104
STEP_REWARD_NAMES = ("foot_frc_score", "foot_vel_score", "orient_cost", "height_error", "step_reward",
                     "upper_body_reward")                                                 # tasks/stepping_task.py:107-120
# held velocity commands (set_command, DESIGN.md §7.6): the WalkingTask envs, and the held flag of the kernel's mode word
# (csrc/sim_core.h MODE_HELD)
COMMAND_ENVS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk")
MODE_HELD = 1 << 30
# chosen footstep plans (reset_footsteps, DESIGN.md §7.7): the SteppingTask's plan types in the order of the kernel's mode word
# (csrc/sim_core.h ST_*)
FOOTSTEP_MODES = ("CURVED", "STANDING", "BACKWARD", "LATERAL", "FORWARD")
# the stair curriculum (stair_curriculum=H, DESIGN.md §7.8): levels of 0.01 m up to H <= 0.2 m (csrc/sim_core.h STAIR_MAX_LEVELS)
STAIR_STEP, STAIR_MAX_HEIGHT = 0.01, 0.2
N_REWARD_SLOTS = 10   # width of the kernel's reward-term record (csrc/sim_core.h NREW); unused slots are 0
# h1_walk (DESIGN.md §4.6): joints (hip_yaw, hip_roll, hip_pitch, knee, ankle), left leg then right.  The mirror swaps the legs and
# negates yaw and roll; in the observation also the root roll and the x, z angular velocities.  The 8 walking-task words map to
# themselves, as in jvrc_walk.  -0.1 stands for "-0" (index 0 negated), as in the reference's lists.
H1_WALK_MIRRORED_OBS = [-0.1, 1, -2, 3, -4,
                        -10, -11, 12, 13, 14, -5, -6, 7, 8, 9,            # joint positions
                        -20, -21, 22, 23, 24, -15, -16, 17, 18, 19,       # joint velocities
                        -30, -31, 32, 33, 34, -25, -26, 27, 28, 29,       # motor torques
                        35, 36, 37, 38, 39, 40, 41, 42]                   # clock sin / cos, mode one-hot, mode reference
H1_WALK_MIRRORED_ACTS = [-5, -6, 7, 8, 9, -0.1, -1, 2, 3, 4]


def push_interval_steps(push_vel: float, push_interval: float, dt: float) -> int:
    """The random pushes' mean interval in control steps, round(push_interval / dt), after refusing a push speed that is
    negative or not finite and an interval that is not finite or shorter than one control step (DESIGN.md §7.5)."""
    push_vel, push_interval = float(push_vel), float(push_interval)
    if not (np.isfinite(push_vel) and push_vel >= 0):
        raise ValueError(f"push_vel must be a finite speed >= 0 m/s, got {push_vel}")
    if not (np.isfinite(push_interval) and push_interval >= dt):
        raise ValueError(f"push_interval must be a finite number of seconds of at least one control step ({dt} s), got {push_interval}")
    return int(round(push_interval / dt))


def stair_levels(model: str, stair_curriculum: float) -> int:
    """The number of levels K = H / 0.01 + 1 of a stair curriculum up to H = stair_curriculum m, or 0 when H is 0 (off), after
    refusing a model other than jvrc_step and an H that is not finite, negative, above 0.2 or not a multiple of 0.01
    (DESIGN.md §7.8)."""
    h = float(stair_curriculum)
    if not np.isfinite(h) or h < 0 or h > STAIR_MAX_HEIGHT:
        raise ValueError(f"stair_curriculum must be a stair height in (0, {STAIR_MAX_HEIGHT:g}] m, or 0 (off), got {stair_curriculum}")
    if h == 0:
        return 0
    k = round(h / STAIR_STEP)
    if abs(k * STAIR_STEP - h) > 1e-9:
        raise ValueError(f"stair_curriculum must be a multiple of {STAIR_STEP:g} m, got {stair_curriculum}")
    if model != "jvrc_step":
        raise ValueError(f"{model} has no stair curriculum: only jvrc_step (SteppingTask) takes one")
    return k + 1


def action_delay_substeps(seconds, sim_dt: float, control_dt: float) -> np.ndarray:
    """Action delays in seconds (a number or a sequence) as whole physics substeps (int32 array), after refusing a value that is
    negative, not finite, above one control step or not a whole number of sim_dt (DESIGN.md §7.9)."""
    s = np.asarray(seconds, dtype=np.float64).reshape(-1)
    bad = ~np.isfinite(s) | (s < 0) | (s > control_dt + 1e-12)
    if bad.any():
        raise ValueError(f"an action delay must lie in [0, {control_dt:g}] s (one control step), got {s[bad][0]}")
    k = np.round(s / sim_dt)
    off = np.abs(k * sim_dt - s) > 1e-9
    if off.any():
        raise ValueError(f"an action delay must be a whole number of physics substeps of {sim_dt:g} s, got {s[off][0]}")
    return k.astype(np.int32)


PAYLOAD_MAX_OFFSET = 0.25   # m: the largest payload offset component (csrc/sim_core.h PAYLOAD_MAX_OFFSET)


def check_payload(mass, offset, total_mass: float) -> tuple[np.ndarray, np.ndarray]:
    """Payload masses (kg, a number or a sequence) and offsets (m, a number or a sequence of numbers or of triples) as float64
    arrays, after refusing a mass that is negative, not finite or above half the robot's total_mass, and an offset component that
    is not finite or whose magnitude is above PAYLOAD_MAX_OFFSET (DESIGN.md §7.10)."""
    m = np.asarray(mass, dtype=np.float64).reshape(-1)
    r = np.asarray(offset, dtype=np.float64)
    bad = ~np.isfinite(m) | (m < 0) | (m > 0.5 * total_mass)
    if bad.any():
        raise ValueError(f"a payload mass must lie in [0, {0.5 * total_mass:g}] kg (half the robot's {total_mass:g} kg), "
                         f"got {m[bad][0]}")
    bad = ~np.isfinite(r) | (np.abs(r) > PAYLOAD_MAX_OFFSET)
    if bad.any():
        raise ValueError(f"a payload offset must lie in [-{PAYLOAD_MAX_OFFSET:g}, {PAYLOAD_MAX_OFFSET:g}] m per axis, "
                         f"got {r[bad].reshape(-1)[0]}")
    return m, r


def check_payload_range(mass: float, offset: float, total_mass: float) -> None:
    """Refuse the random payloads' ranges M (mass U(0, M)) and R (offset U(-R, R)^3) that check_payload refuses as values, a
    negative R, and an R without an M."""
    check_payload(mass, offset, total_mass)
    if offset < 0:
        raise ValueError(f"a payload offset range must be >= 0 m, got {offset}")
    if offset and not mass:
        raise ValueError("a payload offset range needs a payload mass range")


MOTOR_STRENGTH_MAX = 2.0   # the largest motor strength a joint may be given (DESIGN.md §7.11)


def check_motor_strength(strength) -> np.ndarray:
    """Motor strength factors (a number or an array of any shape) as a float64 array of the same shape, after refusing a factor
    that is not finite or lies outside [0, MOTOR_STRENGTH_MAX] (DESIGN.md §7.11)."""
    s = np.asarray(strength, dtype=np.float64)
    bad = ~np.isfinite(s) | (s < 0) | (s > MOTOR_STRENGTH_MAX)
    if bad.any():
        raise ValueError(f"a motor strength must lie in [0, {MOTOR_STRENGTH_MAX:g}], got {s[bad].reshape(-1)[0]}")
    return s


def check_motor_strength_range(max_dev: float) -> None:
    """Refuse the random strengths' range R (every reset draws s ~ U(1 - R, 1 + R) per joint) unless it is finite and in [0, 1]."""
    r = float(max_dev)
    if not (0 <= r <= 1):
        raise ValueError(f"a motor strength range must lie in [0, 1], got {max_dev}")


# sensor errors (DESIGN.md §7.12, csrc/sim_core.h SENSOR_MAX_*): the largest noise multiplier, and the largest roll / pitch (rad),
# gyro (rad/s) and encoder (rad) offsets
SENSOR_MAX_NOISE = 4.0
SENSOR_MAX_BIAS = (0.2, 0.5, 0.2)
SENSOR_BIAS_GROUPS = ("roll / pitch", "gyro", "encoder")


def sensor_bias_bounds(nu: int) -> np.ndarray:
    """The [5 + nu] bounds of an env's offsets, in the order of its sensor row after the multiplier: roll, pitch, gyro x, y, z,
    then the nu motor positions."""
    return np.repeat(np.asarray(SENSOR_MAX_BIAS), [2, 3, nu])


def check_sensor_noise(noise) -> np.ndarray:
    """Noise multipliers (a number or an array of any shape) as a float64 array of the same shape, after refusing one that is not
    finite or lies outside [0, SENSOR_MAX_NOISE] (DESIGN.md §7.12)."""
    m = np.asarray(noise, dtype=np.float64)
    bad = ~np.isfinite(m) | (m < 0) | (m > SENSOR_MAX_NOISE)
    if bad.any():
        raise ValueError(f"a sensor noise multiplier must lie in [0, {SENSOR_MAX_NOISE:g}], got {m[bad].reshape(-1)[0]}")
    return m


def check_sensor_bias(bias, nu: int) -> np.ndarray:
    """Sensor offsets [..., 5 + nu] (roll, pitch, gyro x, y, z, the nu motor positions) as a float64 array, after refusing one that
    is not finite or whose magnitude is above its group's bound of SENSOR_MAX_BIAS."""
    b = np.asarray(bias, dtype=np.float64)
    if b.ndim == 0 or b.shape[-1] != 5 + nu:
        raise ValueError(f"sensor offsets must hold 5 + {nu} = {5 + nu} words per env, got {tuple(b.shape)}")
    bound = sensor_bias_bounds(nu)
    bad = ~np.isfinite(b) | (np.abs(b) > bound)
    if bad.any():
        k = int(np.argwhere(bad)[0][-1])
        g = 0 if k < 2 else 1 if k < 5 else 2
        raise ValueError(f"a {SENSOR_BIAS_GROUPS[g]} offset must lie in [-{SENSOR_MAX_BIAS[g]:g}, {SENSOR_MAX_BIAS[g]:g}], "
                         f"got {b[bad].reshape(-1)[0]}")
    return b


def check_sensor_range(noise: float, bias) -> tuple[float, tuple[float, float, float]]:
    """The random sensor errors' multiplier M and offset ranges (O, G, E) as numbers, after refusing an M that check_sensor_noise
    refuses, a bias that is not three numbers, and a range that is not finite or lies outside [0, its SENSOR_MAX_BIAS bound]."""
    m = float(check_sensor_noise(float(noise)))
    b = np.asarray(bias, dtype=np.float64).reshape(-1)
    if b.shape != (3,):
        raise ValueError(f"a sensor bias range must be three numbers O, G, E (roll / pitch, gyro, encoder), got {bias}")
    for g in range(3):
        if not (0 <= b[g] <= SENSOR_MAX_BIAS[g]):
            raise ValueError(f"a {SENSOR_BIAS_GROUPS[g]} offset range must lie in [0, {SENSOR_MAX_BIAS[g]:g}], got {b[g]}")
    return m, (float(b[0]), float(b[1]), float(b[2]))


class _Robot(SimpleNamespace):
    """The attributes the trainer reads / writes on `env.robot` (robots/robot_base.py:35, run_experiment.py:123-125).
    Writing `iteration_count` (rl/workers/rollout_worker.py:95) drives the SteppingTask's height curriculum."""

    def __setattr__(self, name, value):
        super().__setattr__(name, value)
        if name == "iteration_count" and getattr(self, "_on_iteration", None) is not None:
            self._on_iteration(value)


class BatchedHumanoidEnv:
    def __init__(self, num_envs: int, model: str = "jvrc_walk", precision: int = 32, seed: int = 0,
                 first_env_id: int = 0, device: int | torch.device | None = None, max_traj_len: int = 400,
                 tolerance: float | None = None, max_iter: int | None = None, observation_noise: bool = True,
                 domain_randomization: bool = True, init_noise: bool = True, pd_gain_randomization: float = 0.0,
                 iteration_count: float = float("inf"), path_to_yaml=None, push_vel: float = 0.0, push_interval: float = 15.0,
                 stair_curriculum: float = 0.0, action_delay: float = 0.0, payload_mass: float = 0.0,
                 payload_offset: float = 0.0, motor_strength: float = 0.0, sensor_noise: float = 0.0,
                 sensor_bias=(0.0, 0.0, 0.0)):
        # a stair level per env (DESIGN.md §7.8): every reset builds a FORWARD plan with its level's stair height, and each
        # auto-reset first moves the level by the ending FORWARD episode; off at 0, and then the launches are the plain ones
        self.stair_levels = stair_levels(model, stair_curriculum)
        self.stair_curriculum = float(stair_curriculum) if self.stair_levels else 0.0
        if not torch.cuda.is_available():
            raise _lib.LhwError("BatchedHumanoidEnv needs a CUDA device (no CPU fallback on the rollout path)")
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.num_envs, self.precision, self.seed, self.first_env_id = int(num_envs), int(precision), int(seed), int(first_env_id)
        self.max_traj_len = int(max_traj_len)
        self.dtype = torch.float64 if precision == 64 else torch.float32
        self.model_name = model
        self.mj = load_model(model)
        if path_to_yaml is not None:
            # partial(Env, path_to_yaml) (run_experiment.py:115): the user's YAML over the compiled model's cfg block
            from .config import apply_config, load_yaml
            self.mj = apply_config(self.mj, load_yaml(path_to_yaml))
        self._iteration_count = float(iteration_count)
        # random root-velocity pushes after every control step (DESIGN.md §7.5): off at push_vel == 0, and then nothing is launched
        self.push_vel, self.push_interval = float(push_vel), float(push_interval)
        self.push_interval_steps = push_interval_steps(push_vel, push_interval, self.mj["cfg"]["control_dt"])
        # random action delays (DESIGN.md §7.9): every reset draws its env's delay from U{0 .. action_delay_max} substeps
        self.action_delay_max = int(action_delay_substeps(action_delay, self.mj["cfg"]["sim_dt"], self.mj["cfg"]["control_dt"])[0])
        # random payloads (DESIGN.md §7.10): every reset draws its env's payload, mass U(0, payload_mass), offset
        # U(-payload_offset, payload_offset)^3 on the root link
        check_payload_range(payload_mass, payload_offset, self.mj["total_mass"])
        self.payload_mass, self.payload_offset = float(payload_mass), float(payload_offset)
        # random motor strengths (DESIGN.md §7.11): every reset draws its env's per-joint strengths from U(1 - R, 1 + R)
        check_motor_strength_range(motor_strength)
        self.motor_strength_range = float(motor_strength)
        # random sensor errors (DESIGN.md §7.12): every env observes with noise multiplier sensor_noise, and every reset draws its
        # offsets from U(-O, O) (roll, pitch), U(-G, G) (gyro), U(-E, E) (encoders), sensor_bias = (O, G, E)
        self.sensor_noise, self.sensor_bias = check_sensor_range(sensor_noise, sensor_bias)
        if tolerance is None and precision == 32:
            tolerance = 1e-6  # fp32 cannot reach the reference's 1e-10; gradient floor is ~1e-6 of the force scale
        flat = pack_model(self.mj, tolerance=tolerance, max_iter=max_iter, observation_noise=observation_noise,
                          domain_randomization=domain_randomization, init_noise=init_noise,
                          pd_gain_randomization=pd_gain_randomization, iteration_count=iteration_count)
        L = _lib.lib()
        h = ctypes.c_void_p()
        _lib.check(L.lhw_sim_create(ctypes.byref(h), flat.ctypes.data_as(ctypes.c_void_p), len(flat), self.precision,
                                    self.device.index), "lhw_sim_create")
        self._h = h
        self.obs_dim, self.act_dim = L.lhw_sim_obs_dim(h), L.lhw_sim_act_dim(h)
        n, dev = self.num_envs, self.device
        self.state_r = torch.zeros(n, L.lhw_sim_state_reals(h), dtype=self.dtype, device=dev)
        self.state_i = torch.zeros(n, L.lhw_sim_state_ints(h), dtype=torch.int32, device=dev)
        self.obs = torch.zeros(n, self.obs_dim, dtype=self.dtype, device=dev)
        self.term_obs = torch.zeros(n, self.obs_dim, dtype=self.dtype, device=dev)
        self.reward = torch.zeros(n, dtype=self.dtype, device=dev)
        self.rew_terms = torch.zeros(n, N_REWARD_SLOTS, dtype=self.dtype, device=dev)
        self.done = torch.zeros(n, dtype=torch.int32, device=dev)
        self.ended = torch.zeros(n, dtype=torch.int32, device=dev)
        self.ep_len = torch.zeros(n, dtype=torch.int32, device=dev)
        self.ep_rew = torch.zeros(n, dtype=self.dtype, device=dev)
        self._fresh = True
        # int32 [N]: each env's stair level in [0, stair_levels); None without the curriculum
        self.stair_level = torch.zeros(n, dtype=torch.int32, device=dev) if self.stair_levels else None
        # int32 [N]: each env's action delay in physics substeps; None (and the plain step kernels) until random delays or
        # set_action_delay create it
        self.action_delay = torch.zeros(n, dtype=torch.int32, device=dev) if self.action_delay_max else None
        # [N, 4] of the env's dtype: each env's payload (m, rx, ry, rz); None (and the plain step kernels) until random payloads or
        # set_payload create it
        self.payload = torch.zeros(n, 4, dtype=self.dtype, device=dev) if self.payload_mass else None
        # [N, act_dim] of the env's dtype: each env's motor strengths; None (and the launches without them) until random strengths
        # or set_motor_strength create it
        self.motor_strength = (torch.ones(n, self.act_dim, dtype=self.dtype, device=dev) if self.motor_strength_range else None)
        # [N, 6 + act_dim] of the env's dtype: each env's noise multiplier, then its offsets (roll, pitch, gyro x, y, z, the motor
        # positions); None (and no sensor pass) until random sensor errors or set_sensor_errors create it
        self.sensor = None
        if self.sensor_noise or any(self.sensor_bias):
            self.sensor = torch.zeros(n, 6 + self.act_dim, dtype=self.dtype, device=dev)
            self.sensor[:, 0] = self.sensor_noise
        # ---- reference-facing attributes (envs/jvrc/jvrc_base.py:69-131, envs/jvrc/jvrc_walk.py:43-63)
        cfg = self.mj["cfg"]
        self.history_len = cfg["obs_history_len"]
        self.base_obs_len = self.obs_dim
        self.dt = cfg["control_dt"]
        self.action_space = np.zeros(self.act_dim)
        self.observation_space = np.zeros(self.obs_dim * self.history_len)
        self.nq, self.nv = 7 + self.act_dim, 6 + self.act_dim
        self._setup_reference_attributes(model, cfg)
        # env.interface / env.task / env.model / env.data of the reference's env protocol (SURVEY.md §8b), as views of env 0
        from ..tasks.descriptors import DataView, DeviceRobotInterface, make_task, model_view
        self.interface = DeviceRobotInterface(self, 0)
        self.task = make_task(self, 0)
        self.model, self.data = model_view(self), DataView(self, 0)

    def _setup_reference_attributes(self, model: str, cfg: dict) -> None:
        """obs_mean / obs_std, reward names and the robot's mirror lists exactly as the reference env classes set them
        (pure numpy; pinned to the reference's own method bodies by tests/golden/env_attributes.json)."""
        if model in ("h1", "h1_walk"):
            # envs/h1/h1_env.py:37-55 (normalisation), envs/h1/h1_base.py:66-76 ; no mirror lists on the H1 robot
            self.reward_names = STAND_REWARD_NAMES
            half = np.asarray(cfg["half_sitting_pose"], dtype=float)
            self.obs_mean = np.concatenate((np.zeros(5), half, np.zeros(10), np.zeros(10)))
            self.obs_std = np.concatenate(([0.2, 0.2, 1, 1, 1], 0.5 * np.ones(10), 4 * np.ones(10), 100 * np.ones(10)))
            self.robot = SimpleNamespace(iteration_count=np.inf)
            if model == "h1":
                return
            # h1_walk: h1's 35 robot-state entries, then jvrc_walk's 8 walking-task words (clock, mode one-hot, reference)
            self.reward_names = REWARD_NAMES
            self.obs_mean = np.concatenate((self.obs_mean, [0, 0, 0.5, 0.5, 0.5, 0, 0, 0]))
            self.obs_std = np.concatenate((self.obs_std, [1, 1, 1, 1, 1, 0.5, 0.5, 0.5]))
            self.robot = _Robot(mirrored_obs=list(H1_WALK_MIRRORED_OBS), mirrored_acts=list(H1_WALK_MIRRORED_ACTS),
                                clock_inds=[35, 36], iteration_count=self._iteration_count, _on_iteration=None)
            return
        self.reward_names = REWARD_NAMES
        half = np.deg2rad(cfg["half_sitting_pose_deg"])
        self.obs_mean = np.concatenate((np.zeros(5), half, np.zeros(12), [0, 0, 0.5, 0.5, 0.5, 0, 0, 0]))
        self.obs_std = np.concatenate(([0.2, 0.2, 1, 1, 1], 0.5 * np.ones(12), 4 * np.ones(12), [1, 1, 1, 1, 1, 0.5, 0.5, 0.5]))
        base_mir_obs = [-0.1, 1, -2, 3, -4, 11, -12, -13, 14, -15, 16, 5, -6, -7, 8, -9, 10,
                        23, -24, -25, 26, -27, 28, 17, -18, -19, 20, -21, 22]
        append_obs = [len(base_mir_obs) + i for i in range(8)]
        if model not in ("jvrc_walk", "jvrc_walk_terrain", "jvrc_step"):
            raise ValueError(f"unknown model {model!r}")
        if model == "jvrc_step":
            # envs/jvrc/jvrc_step.py:41-63: clock(2) + goal steps x(2) y(2) z(2) theta(2)
            self.reward_names = STEP_REWARD_NAMES
            self.obs_mean = np.concatenate((np.zeros(5), half, np.zeros(12), [0.5, 0.5], np.zeros(8)))
            self.obs_std = np.concatenate(([0.2, 0.2, 1, 1, 1], 0.5 * np.ones(12), 4 * np.ones(12), [1, 1], np.ones(8)))
            append_obs = [len(base_mir_obs) + i for i in range(10)]
        self.robot = _Robot(mirrored_obs=base_mir_obs + append_obs,
                            mirrored_acts=[6, -7, -8, 9, -10, 11, 0.1, -1, -2, 3, -4, 5],
                            clock_inds=append_obs[0:2], iteration_count=self._iteration_count, _on_iteration=None)
        if model == "jvrc_step":
            self.robot._on_iteration = self._set_iteration_count

    def _set_iteration_count(self, iteration_count: float) -> None:
        """SteppingTask.reset(iter_count) (tasks/stepping_task.py:262-264, 312): the curriculum's step height for the
        episodes that start from now on."""
        _lib.check(_lib.lib().lhw_sim_set_step_height(self._h, float(curriculum_height(iteration_count))),
                   "lhw_sim_set_step_height")

    # ------------------------------------------------------------------ device API (torch tensors in / out)
    def reset(self, mask: torch.Tensor | None = None) -> torch.Tensor:
        """Reset all envs (or those where mask != 0); returns the [N, obs_dim] observation tensor."""
        L = _lib.lib()
        if mask is not None:
            mask = mask.to(device=self.device, dtype=torch.int32).contiguous()
        if self.stair_level is not None:
            _lib.ops().sim_reset_stairs(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id, mask,
                                        bool(self._fresh and mask is None), self.obs, self.stair_level, self.stair_levels)
        elif _lib.use_torch_ops():
            _lib.ops().sim_reset(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id, mask,
                                 bool(self._fresh and mask is None), self.obs)
        else:
            with torch.cuda.device(self.device):
                _lib.check(L.lhw_sim_reset(self._h, self.state_r.data_ptr(), self.state_i.data_ptr(), self.num_envs, self.seed,
                                           self.first_env_id, _lib.ptr(mask), int(self._fresh and mask is None),
                                           self.obs.data_ptr(), _lib.current_stream_ptr()), "lhw_sim_reset")
        if mask is None:
            self._fresh = False
        self._draw_delay(0, self.num_envs, mask)
        self._draw_payload(0, self.num_envs, mask)
        self._draw_motor(0, self.num_envs, mask)
        self._sense(0, self.num_envs, mask, False, False)
        return self.obs

    def step(self, actions: torch.Tensor, autoreset: bool = True):
        """actions [N, act_dim] (device, env dtype). Returns (obs, reward, done, ended) device tensors.
        With autoreset the RolloutWorker semantics apply (see include/lhw_b200.h: lhw_sim_step)."""
        if actions.dtype != self.dtype or not actions.is_contiguous() or actions.device != self.device:
            actions = actions.to(device=self.device, dtype=self.dtype).contiguous()
        if self.motor_strength is not None:
            self._step_motor(0, self.num_envs, actions, autoreset)
            self._sense(0, self.num_envs, self.ended, True, autoreset)
            return self.obs, self.reward, self.done, self.ended
        if self.payload is not None:
            self._step_payload(0, self.num_envs, actions, autoreset)
            self._sense(0, self.num_envs, self.ended, True, autoreset)
            return self.obs, self.reward, self.done, self.ended
        if self.action_delay is not None:
            self._step_delay(0, self.num_envs, actions, autoreset)
            self._sense(0, self.num_envs, self.ended, True, autoreset)
            return self.obs, self.reward, self.done, self.ended
        if self.stair_level is not None:
            _lib.ops().sim_step_stairs(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id, actions, self.max_traj_len,
                                       bool(autoreset), self.obs, self.term_obs, self.reward, self.rew_terms, self.done, self.ended,
                                       self.ep_len, self.ep_rew, self.stair_level, self.stair_levels)
            self._push_random(0, self.num_envs)
            self._sense(0, self.num_envs, self.ended, True, autoreset)
            return self.obs, self.reward, self.done, self.ended
        if _lib.use_torch_ops():     # torch.ops.lhw.sim_step: device / dtype / shape checks, then the C-ABI launch
            _lib.ops().sim_step(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id, actions, self.max_traj_len,
                                bool(autoreset), self.obs, self.term_obs, self.reward, self.rew_terms, self.done, self.ended,
                                self.ep_len, self.ep_rew)
            self._push_random(0, self.num_envs)
            self._sense(0, self.num_envs, self.ended, True, autoreset)
            return self.obs, self.reward, self.done, self.ended
        assert actions.shape == (self.num_envs, self.act_dim), actions.shape
        L = _lib.lib()
        with torch.cuda.device(self.device):
            _lib.check(L.lhw_sim_step(self._h, self.state_r.data_ptr(), self.state_i.data_ptr(), self.num_envs, self.seed,
                                      self.first_env_id, actions.data_ptr(), self.max_traj_len, int(autoreset),
                                      self.obs.data_ptr(), self.term_obs.data_ptr(), self.reward.data_ptr(),
                                      self.rew_terms.data_ptr(), self.done.data_ptr(), self.ended.data_ptr(),
                                      self.ep_len.data_ptr(), self.ep_rew.data_ptr(), _lib.current_stream_ptr()),
                       "lhw_sim_step")
        self._push_random(0, self.num_envs)
        self._sense(0, self.num_envs, self.ended, True, autoreset)
        return self.obs, self.reward, self.done, self.ended

    def step_slice(self, lo: int, hi: int, actions: torch.Tensor, autoreset: bool = True):
        """One control step of environments [lo, hi) only (their records, outputs and Philox ids are the same as in a full-batch
        step: an environment's trajectory does not depend on what it is launched with).  The rollout worker advances two halves
        of the batch on two streams with this, so that the tail of one half's launch overlaps the other half's work."""
        sl = slice(lo, hi)
        if actions.dtype != self.dtype or not actions.is_contiguous() or actions.device != self.device:
            actions = actions.to(device=self.device, dtype=self.dtype).contiguous()
        out = (self.obs[sl], self.reward[sl], self.done[sl], self.ended[sl])
        if self.motor_strength is not None:
            self._step_motor(lo, hi, actions, autoreset)
            self._sense(lo, hi, out[3], True, autoreset)
            return out
        if self.payload is not None:
            self._step_payload(lo, hi, actions, autoreset)
            self._sense(lo, hi, out[3], True, autoreset)
            return out
        if self.action_delay is not None:
            self._step_delay(lo, hi, actions, autoreset)
            self._sense(lo, hi, out[3], True, autoreset)
            return out
        if self.stair_level is not None:
            _lib.ops().sim_step_stairs(self._h.value, self.state_r[sl], self.state_i[sl], self.seed, self.first_env_id + lo, actions,
                                       self.max_traj_len, bool(autoreset), out[0], self.term_obs[sl], out[1], self.rew_terms[sl], out[2],
                                       out[3], self.ep_len[sl], self.ep_rew[sl], self.stair_level[sl], self.stair_levels)
            self._push_random(lo, hi)
            self._sense(lo, hi, out[3], True, autoreset)
            return out
        if _lib.use_torch_ops():
            _lib.ops().sim_step(self._h.value, self.state_r[sl], self.state_i[sl], self.seed, self.first_env_id + lo, actions,
                                self.max_traj_len, bool(autoreset), out[0], self.term_obs[sl], out[1], self.rew_terms[sl], out[2], out[3],
                                self.ep_len[sl], self.ep_rew[sl])
            self._push_random(lo, hi)
            self._sense(lo, hi, out[3], True, autoreset)
            return out
        assert actions.shape == (hi - lo, self.act_dim), actions.shape
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().lhw_sim_step(self._h, self.state_r[sl].data_ptr(), self.state_i[sl].data_ptr(), hi - lo, self.seed,
                                               self.first_env_id + lo, actions.data_ptr(), self.max_traj_len, int(autoreset),
                                               out[0].data_ptr(), self.term_obs[sl].data_ptr(), out[1].data_ptr(),
                                               self.rew_terms[sl].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                               self.ep_len[sl].data_ptr(), self.ep_rew[sl].data_ptr(), _lib.current_stream_ptr()),
                       "lhw_sim_step")
        self._push_random(lo, hi)
        self._sense(lo, hi, out[3], True, autoreset)
        return out

    def _step_delay(self, lo: int, hi: int, actions: torch.Tensor, autoreset: bool) -> None:
        """The delayed control step of environments [lo, hi) (with the stair curriculum when it is on), then, in random mode and
        with autoreset, the delay draw of the envs it ended (and so reset), then the random pushes; all on the current stream."""
        sl = slice(lo, hi)
        level = None if self.stair_level is None else self.stair_level[sl]
        _lib.ops().sim_step_delay(self._h.value, self.state_r[sl], self.state_i[sl], self.seed, self.first_env_id + lo, actions,
                                  self.max_traj_len, bool(autoreset), self.obs[sl], self.term_obs[sl], self.reward[sl], self.rew_terms[sl],
                                  self.done[sl], self.ended[sl], self.ep_len[sl], self.ep_rew[sl], self.action_delay[sl], level,
                                  self.stair_levels)
        if autoreset:
            self._draw_delay(lo, hi, self.ended[sl])
        self._push_random(lo, hi)

    def _draw_delay(self, lo: int, hi: int, mask: torch.Tensor | None) -> None:
        """Random mode: environments [lo, hi) whose mask word is non-zero (all without a mask), just reset, draw their new
        episode's delay; nothing is launched otherwise (include/lhw_b200.h: lhw_sim_draw_delay)."""
        if self.action_delay_max:
            _lib.ops().sim_draw_delay(self._h.value, self.state_i[lo:hi], self.seed, self.first_env_id + lo, mask, self.action_delay_max,
                                      self.action_delay[lo:hi])

    def set_action_delay(self, seconds) -> None:
        """Give every environment an action delay: seconds holds N values (a sequence or tensor), each a whole number of physics
        substeps in [0, control_dt].  In a control step, the first delay / sim_dt substeps still drive the PD loop towards the
        previous step's target.  The delays hold until each env's next reset draws a new one (random mode, action_delay > 0) or
        until they are set again (include/lhw_b200.h: lhw_sim_step_delay)."""
        s = torch.as_tensor(seconds, dtype=torch.float64).detach().to("cpu").reshape(-1)
        if s.shape != (self.num_envs,):
            raise ValueError(f"seconds must hold {self.num_envs} numbers, got {tuple(s.shape)}")
        d = action_delay_substeps(s.numpy(), self.mj["cfg"]["sim_dt"], self.mj["cfg"]["control_dt"])
        if self.action_delay is None:
            self.action_delay = torch.zeros(self.num_envs, dtype=torch.int32, device=self.device)
        self.action_delay.copy_(torch.from_numpy(d))

    def _step_payload(self, lo: int, hi: int, actions: torch.Tensor, autoreset: bool) -> None:
        """The control step of environments [lo, hi) with their payloads (and their action delays and stair levels when those
        are on), then, with autoreset, the random draws of the envs it ended (and so reset), then the random pushes; all on the
        current stream."""
        sl = slice(lo, hi)
        delay = None if self.action_delay is None else self.action_delay[sl]
        level = None if self.stair_level is None else self.stair_level[sl]
        _lib.ops().sim_step_payload(self._h.value, self.state_r[sl], self.state_i[sl], self.seed, self.first_env_id + lo, actions,
                                    self.max_traj_len, bool(autoreset), self.obs[sl], self.term_obs[sl], self.reward[sl],
                                    self.rew_terms[sl], self.done[sl], self.ended[sl], self.ep_len[sl], self.ep_rew[sl],
                                    self.payload[sl], delay, level, self.stair_levels)
        if autoreset:
            self._draw_delay(lo, hi, self.ended[sl])
            self._draw_payload(lo, hi, self.ended[sl])
        self._push_random(lo, hi)

    def _draw_payload(self, lo: int, hi: int, mask: torch.Tensor | None) -> None:
        """Random mode: environments [lo, hi) whose mask word is non-zero (all without a mask), just reset, draw their new
        episode's payload; nothing is launched otherwise (include/lhw_b200.h: lhw_sim_draw_payload)."""
        if self.payload_mass:
            _lib.ops().sim_draw_payload(self._h.value, self.state_i[lo:hi], self.seed, self.first_env_id + lo, mask, self.payload_mass,
                                        self.payload_offset, self.payload[lo:hi])

    def set_payload(self, mass, offset=None) -> None:
        """Give every environment a payload on its root link: mass holds N values in kg (a sequence or tensor), offset None (at
        the root link's centre of mass), one (x, y, z) for every env or [N, 3], in m in the root link's frame relative to the
        compiled model's root-link centre of mass.  A mass is at most half the robot's total_mass, an offset component at most
        0.25 m in magnitude.  The payloads hold until each env's next reset draws a new one (random mode, payload_mass > 0) or
        until they are set again (include/lhw_b200.h: lhw_sim_step_payload)."""
        m = torch.as_tensor(mass, dtype=torch.float64).detach().to("cpu").reshape(-1)
        if m.shape != (self.num_envs,):
            raise ValueError(f"mass must hold {self.num_envs} numbers, got {tuple(m.shape)}")
        r = np.zeros(3) if offset is None else torch.as_tensor(offset, dtype=torch.float64).detach().to("cpu").numpy()
        if r.shape not in ((3,), (self.num_envs, 3)):
            raise ValueError(f"offset must be (x, y, z) or [{self.num_envs}, 3], got {tuple(r.shape)}")
        m, r = check_payload(m.numpy(), r, self.mj["total_mass"])
        host = np.concatenate([m[:, None], np.broadcast_to(r, (self.num_envs, 3))], axis=1)
        if self.payload is None:
            self.payload = torch.zeros(self.num_envs, 4, dtype=self.dtype, device=self.device)
        self.payload.copy_(torch.from_numpy(host))

    def _step_motor(self, lo: int, hi: int, actions: torch.Tensor, autoreset: bool) -> None:
        """The control step of environments [lo, hi) with their motor strengths (and their payloads, action delays and stair levels
        when those are on), then, with autoreset, the random draws of the envs it ended (and so reset), then the random pushes; all
        on the current stream."""
        sl = slice(lo, hi)
        payload = None if self.payload is None else self.payload[sl]
        delay = None if self.action_delay is None else self.action_delay[sl]
        level = None if self.stair_level is None else self.stair_level[sl]
        _lib.ops().sim_step_motor(self._h.value, self.state_r[sl], self.state_i[sl], self.seed, self.first_env_id + lo, actions,
                                  self.max_traj_len, bool(autoreset), self.obs[sl], self.term_obs[sl], self.reward[sl], self.rew_terms[sl],
                                  self.done[sl], self.ended[sl], self.ep_len[sl], self.ep_rew[sl], self.motor_strength[sl], payload, delay,
                                  level, self.stair_levels)
        if autoreset:
            self._draw_delay(lo, hi, self.ended[sl])
            self._draw_payload(lo, hi, self.ended[sl])
            self._draw_motor(lo, hi, self.ended[sl])
        self._push_random(lo, hi)

    def _draw_motor(self, lo: int, hi: int, mask: torch.Tensor | None) -> None:
        """Random mode: environments [lo, hi) whose mask word is non-zero (all without a mask), just reset, draw their new
        episode's motor strengths; nothing is launched otherwise (include/lhw_b200.h: lhw_sim_draw_motor)."""
        if self.motor_strength_range:
            _lib.ops().sim_draw_motor(self._h.value, self.state_i[lo:hi], self.seed, self.first_env_id + lo, mask,
                                      self.motor_strength_range, self.motor_strength[lo:hi])

    def set_motor_strength(self, strength) -> None:
        """Give every environment's actuated joints a motor strength: strength is [N, act_dim] (one factor per env and joint, in
        get_motor_names() order) or [N] (one factor for all of an env's joints), each in [0, 2].  Joint l then delivers
        s_l (kp (target - q) + kd (0 - qdot)).  The strengths hold until each env's next reset draws new ones (random mode,
        motor_strength > 0) or until they are set again (include/lhw_b200.h: lhw_sim_step_motor)."""
        s = torch.as_tensor(strength, dtype=torch.float64).detach().to("cpu")
        if s.shape == (self.num_envs,):
            s = s[:, None].expand(self.num_envs, self.act_dim)
        if s.shape != (self.num_envs, self.act_dim):
            raise ValueError(f"strength must be [{self.num_envs}, {self.act_dim}] or [{self.num_envs}], got {tuple(s.shape)}")
        host = check_motor_strength(s.numpy())
        if self.motor_strength is None:
            self.motor_strength = torch.ones(self.num_envs, self.act_dim, dtype=self.dtype, device=self.device)
        self.motor_strength.copy_(torch.from_numpy(np.ascontiguousarray(host)))

    def _sense(self, lo: int, hi: int, sel: torch.Tensor | None, after_step: bool, autoreset: bool) -> None:
        """The sensor errors of environments [lo, hi), on the current stream after the launches that wrote their observations;
        nothing is launched while self.sensor is None.  After a step (sel: its ended flags), with autoreset an env that ended gets
        the ending episode's errors on its term_obs, draws its new offsets (random mode) and gets them on its obs; every other obs
        gets its env's errors, and without autoreset term_obs the same.  After a reset (sel: its mask, None for every env) the
        selected envs draw (random mode) and get them on their obs (include/lhw_b200.h: lhw_sim_sense)."""
        if self.sensor is None:
            return
        draw = list(self.sensor_bias) if any(self.sensor_bias) else None
        _lib.ops().sim_sense(self._h.value, self.state_i[lo:hi], self.seed, self.first_env_id + lo, sel, bool(after_step),
                             bool(autoreset), draw, self.sensor[lo:hi], self.obs[lo:hi], self.term_obs[lo:hi] if after_step else None)

    def set_sensor_errors(self, noise, bias=None) -> None:
        """Give every environment sensor errors: noise is one multiplier m or N of them, in [0, 4]; bias None (no offsets), one row
        of 5 + act_dim offsets for every env or [N, 5 + act_dim]: roll and pitch (rad, at most 0.2), gyro x, y, z (rad/s, at most
        0.5) and one per motor position (rad, at most 0.2, in get_motor_names() order).  Each observed robot-state word then gets
        its offset plus m times its group's noise scale times U(-1, 1).  The errors hold until each env's next random draw (random
        mode) or until they are set again; the current obs is not rewritten, so errors set before a reset apply from that reset's
        observation on (include/lhw_b200.h: lhw_sim_sense)."""
        n, nb = self.num_envs, 5 + self.act_dim
        m = torch.as_tensor(noise, dtype=torch.float64).detach().to("cpu").reshape(-1)
        if m.shape == (1,):
            m = m.expand(n)
        if m.shape != (n,):
            raise ValueError(f"noise must be one number or {n}, got {tuple(m.shape)}")
        b = np.zeros((n, nb)) if bias is None else torch.as_tensor(bias, dtype=torch.float64).detach().to("cpu").numpy()
        if b.shape == (nb,):
            b = np.broadcast_to(b, (n, nb))
        if b.shape != (n, nb):
            raise ValueError(f"bias must be None, [{nb}] or [{n}, {nb}], got {tuple(b.shape)}")
        host = np.concatenate([check_sensor_noise(m.numpy())[:, None], check_sensor_bias(b, self.act_dim)], axis=1)
        if self.sensor is None:
            self.sensor = torch.zeros(n, 6 + self.act_dim, dtype=self.dtype, device=self.device)
        self.sensor.copy_(torch.from_numpy(host))

    def _push_random(self, lo: int, hi: int) -> None:
        """The random pushes of environments [lo, hi) after their control step, on the same stream; none at push_vel == 0.
        An env that the step ended (and so reset) is not pushed; the draws are keyed by the env's Philox id and event counter."""
        if self.push_vel > 0:
            _lib.ops().sim_push(self._h.value, self.state_r[lo:hi], self.state_i[lo:hi], self.seed, self.first_env_id + lo,
                                self.ended[lo:hi], self.push_vel, self.push_interval_steps, None)

    def push(self, d: torch.Tensor) -> None:
        """Push every environment once, now: d [N, 2] holds each one's velocity change (dx, dy) in m/s in its heading frame (x
        forward, y to the robot's left), added to the root's world-frame qvel[0:2] after rotation by the heading.  Rows that are
        exactly zero are left untouched, and nothing else of any record changes (include/lhw_b200.h: lhw_sim_push)."""
        if d.dtype != self.dtype or not d.is_contiguous() or d.device != self.device:
            d = d.to(device=self.device, dtype=self.dtype).contiguous()
        _lib.ops().sim_push(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id, None, 0.0, 1, d)

    def set_command(self, mode, ref) -> None:
        """Give environments a velocity command and hold it until each one's next reset: mode [N] holds per env -1 (untouched),
        0 (STANDING), 1 (INPLACE) or 2 (FORWARD), and ref [N, 3] its reference (yaw_rate rad/s, vx m/s, vy m/s), in the order of the
        record's mode_ref; sequences or tensors.  The WalkingTask's random mode switches skip a held env, and the six task words of
        self.obs are rewritten, so the next action already sees the command (include/lhw_b200.h: lhw_sim_set_command).  Values
        outside the training ranges (DESIGN.md §7.6) are accepted; non-finite ones and other modes are refused."""
        if self.model_name not in COMMAND_ENVS:
            raise ValueError(f"{self.model_name} has no velocity command: only the WalkingTask envs {', '.join(COMMAND_ENVS)} take one")
        mode = torch.as_tensor(mode).detach().to("cpu").reshape(-1)
        ref = torch.as_tensor(ref, dtype=torch.float64).detach().to("cpu")
        if mode.dtype.is_floating_point or mode.dtype == torch.bool or mode.shape != (self.num_envs,):
            raise ValueError(f"mode must hold {self.num_envs} integers, got {tuple(mode.shape)} of {mode.dtype}")
        if ref.shape != (self.num_envs, 3):
            raise ValueError(f"ref must be [{self.num_envs}, 3] (yaw_rate, vx, vy), got {tuple(ref.shape)}")
        if ((mode < -1) | (mode > 2)).any():
            raise ValueError(f"mode must be -1 (untouched), 0 (STANDING), 1 (INPLACE) or 2 (FORWARD), got {sorted(set(mode.tolist()))}")
        if not torch.isfinite(ref).all():
            raise ValueError("ref must be finite")
        _lib.ops().sim_set_command(self._h.value, self.state_r, self.state_i, mode.to(device=self.device, dtype=torch.int32),
                                   ref.to(device=self.device, dtype=self.dtype), self.obs)

    def footstep_limits(self) -> tuple[int, float]:
        """(number of curved plans, largest FORWARD stair height |h| in m) that reset_footsteps accepts: the plans of
        model/jvrc_step.json, and twice a slab's half height (above it a slab's side face no longer covers the riser below the next
        slab)."""
        if self.model_name != "jvrc_step":
            raise ValueError(f"{self.model_name} has no footstep plan: only jvrc_step (SteppingTask) takes one")
        st = self.mj["stepping"]
        return len(st["plans"]), 2 * float(st["slab_half"][2])

    def reset_footsteps(self, mode, value) -> torch.Tensor:
        """Reset environments with a chosen stepping-stone plan; returns self.obs.  mode [N] holds per env -1 (untouched) or a plan
        type of FOOTSTEP_MODES (0 CURVED, 1 STANDING, 2 BACKWARD, 3 LATERAL, 4 FORWARD), value [N] its value: FORWARD the signed
        stair height in m, LATERAL +1 (to the robot's left) or -1, CURVED a plan index or -1 (the reset's own draw), STANDING and
        BACKWARD 0; sequences or tensors.  Every other draw of the reset is the plain reset's, and the plan lasts for the episode
        (include/lhw_b200.h: lhw_sim_reset_footsteps).  On a fresh env every row needs a plan."""
        nplan, max_h = self.footstep_limits()
        mode = torch.as_tensor(mode).detach().to("cpu").reshape(-1)
        value = torch.as_tensor(value, dtype=torch.float64).detach().to("cpu").reshape(-1)
        if mode.dtype.is_floating_point or mode.dtype == torch.bool or mode.shape != (self.num_envs,):
            raise ValueError(f"mode must hold {self.num_envs} integers, got {tuple(mode.shape)} of {mode.dtype}")
        if value.shape != (self.num_envs,):
            raise ValueError(f"value must hold {self.num_envs} numbers, got {tuple(value.shape)}")
        if ((mode < -1) | (mode > 4)).any():
            raise ValueError(f"mode must be -1 (untouched) or 0..4 ({', '.join(FOOTSTEP_MODES)}), got {sorted(set(mode.tolist()))}")
        if not torch.isfinite(value).all():
            raise ValueError("value must be finite")
        if ((mode == 4) & (value.abs() > max_h)).any():
            raise ValueError(f"a FORWARD stair height must lie in [-{max_h:g}, {max_h:g}] m")
        if ((mode == 3) & (value != 1) & (value != -1)).any():
            raise ValueError("a LATERAL value must be +1 (left) or -1 (right)")
        if ((mode == 0) & (value != -1) & ((value < 0) | (value >= nplan) | (value != value.floor()))).any():
            raise ValueError(f"a CURVED value must be -1 (drawn) or a plan index in [0, {nplan})")
        if (((mode == 1) | (mode == 2)) & (value != 0)).any():
            raise ValueError("a STANDING or BACKWARD value must be 0")
        if self._fresh and (mode < 0).any():
            raise ValueError("this env has never been reset: give every row a plan, or call reset() first")
        _lib.ops().sim_reset_footsteps(self._h.value, self.state_r, self.state_i, self.seed, self.first_env_id,
                                       mode.to(device=self.device, dtype=torch.int32), value.to(device=self.device, dtype=self.dtype),
                                       self._fresh, self.obs)
        self._fresh = False
        if self.action_delay_max or self.payload_mass or self.motor_strength_range:
            picked = (mode >= 0).to(device=self.device, dtype=torch.int32)
            self._draw_delay(0, self.num_envs, picked)
            self._draw_payload(0, self.num_envs, picked)
            self._draw_motor(0, self.num_envs, picked)
        if self.sensor is not None:
            self._sense(0, self.num_envs, (mode >= 0).to(device=self.device, dtype=torch.int32), False, False)
        return self.obs

    def command_accumulate(self, acc: torch.Tensor) -> torch.Tensor:
        """Add the last control step (taken with autoreset=False) to the command sweep's signed-velocity records acc, a
        zero-initialised [N, command_words()] float64 device tensor: steps, the sums of v_fwd, v_lat and w_z, ended-by-done, over
        the steps eval_accumulate counts (include/lhw_b200.h: lhw_sim_command_accumulate)."""
        _lib.ops().sim_command_accumulate(self._h.value, self.state_r, self.done, acc)
        return acc

    @staticmethod
    def command_words() -> int:
        return _lib.lib().lhw_sim_command_words()

    def eval_accumulate(self, acc: torch.Tensor) -> torch.Tensor:
        """Add the last control step (taken with autoreset=False) to the evaluation accumulators acc, a zero-initialised
        [N, eval_words()] float64 device tensor, in one launch that only reads the step's outputs and the records (include/lhw_b200.h:
        lhw_sim_eval_accumulate; rl/evaluation.py names the words)."""
        _lib.ops().sim_eval_accumulate(self._h.value, self.state_r, self.state_i, self.reward, self.rew_terms, self.done, acc)
        return acc

    @staticmethod
    def eval_words() -> int:
        return _lib.lib().lhw_sim_eval_words()

    def bind(self):
        """Upload this env's model constants if another env of the same precision used the constant bank last
        (needed before replaying CUDA graphs that contain lhw_sim_step launches)."""
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().lhw_sim_bind(self._h, _lib.current_stream_ptr()), "lhw_sim_bind")

    def render_rgb(self, env_ids=(0,), width: int = 640, height: int = 480) -> torch.Tensor:
        """Pictures of environments env_ids as a device uint8 tensor [len(env_ids), height, width, 3] (RGB, row 0 at the top),
        ray-cast in one launch from their current records, which are only read.  The tracking camera looks at each robot from
        the side (from -y), 3 m away, 15 degrees down, with a 45 degree vertical field of view (include/lhw_b200.h:
        lhw_sim_render).  What is drawn: csrc/render_core.h."""
        ids = torch.as_tensor(env_ids, dtype=torch.int32).reshape(-1).to(self.device)
        rgb = torch.empty(len(ids), height, width, 3, dtype=torch.uint8, device=self.device)
        cam = (0.0, 0.0, 0.9 if self.model_name in ("h1", "h1_walk") else 0.8, 3.0, 90.0, 15.0, 45.0)   # dx dy z distance azimuth elevation fovy
        if _lib.use_torch_ops():
            _lib.ops().sim_render(self._h.value, self.state_r, self.state_i, ids, width, height, *cam, rgb)
            return rgb
        if len(ids) and not (0 <= int(ids.min()) and int(ids.max()) < self.num_envs):
            raise ValueError(f"env_ids must lie in [0, {self.num_envs})")
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().lhw_sim_render(self._h, self.state_r.data_ptr(), self.state_i.data_ptr(), self.num_envs, ids.data_ptr(),
                                                 len(ids), width, height, *cam, rgb.data_ptr(), _lib.current_stream_ptr()),
                       "lhw_sim_render")
        return rgb

    # ------------------------------------------------------------------ host API (numpy in / out, copies inside)
    def step_host(self, actions: np.ndarray, autoreset: bool = True):
        """Reference-facing batched call with HOST buffers: H2D actions, one launch, D2H obs/reward/done."""
        a = torch.from_numpy(np.ascontiguousarray(actions, dtype=np.float64 if self.precision == 64 else np.float32))
        obs, rew, done, ended = self.step(a.to(self.device, non_blocking=True), autoreset)
        return obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy().astype(bool), ended.cpu().numpy().astype(bool)

    # ------------------------------------------------------------------ state access (tests / checkpointing)
    @property
    def qpos(self) -> torch.Tensor:
        return self.state_r[:, 0:self.nq]

    @property
    def qvel(self) -> torch.Tensor:
        return self.state_r[:, self.nq:self.nq + self.nv]

    def solver_iterations(self) -> torch.Tensor:
        """Newton iterations spent in the last launch, per env."""
        return self.state_i[:, 7]

    def status_flags(self) -> torch.Tensor:
        """Per-env status word of the last launch (1: non-finite / diverging acceleration seen, forced reset — the analogue
        of MuJoCo's mj_checkAcc auto-reset; 2: a Cholesky pivot had to be clamped)."""
        return self.state_i[:, 6]

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            _lib.lib().lhw_sim_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
