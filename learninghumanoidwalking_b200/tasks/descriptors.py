"""Host-side task descriptors and the RobotInterface-style view over the device state (SURVEY.md §8b "Task protocol",
"Env protocol": env.task, env.interface, env.model, env.data).

`WalkingTask` / `SteppingTask` / `StandingTask` subclass BaseTask and keep the reference's attribute names
(tasks/walking_task.py:45-84, tasks/stepping_task.py:26-50, tasks/standing_task.py:14-47): `_goal_height_ref`,
`_swing_duration`, `_stance_duration`, `_total_duration`, `_neutral_pose`, `_mass`, `_root_body_name`, ...; plus `weights`,
the reward-term weights the kernel applies.  Their hooks read back what the kernel did for environment `index` of the batch.
`DeviceRobotInterface` offers the getters of envs/common/robot_interface.py that can be answered from the per-env state
record (qpos, qvel, qacc, the LAGGED actuator state the PD law and the observation use, last joint torques)."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from .base_task import BaseTask

WALK_WEIGHTS = dict(foot_frc_score=0.225, foot_vel_score=0.225, root_accel=0.050, height_error=0.050, com_vel_error=0.150,
                    yaw_vel_error=0.150, upper_body_reward=0.050, posture_error=0.050, torque_penalty=0.025,
                    action_penalty=0.025)                                            # tasks/walking_task.py:131-146
STEP_WEIGHTS = dict(foot_frc_score=0.150, foot_vel_score=0.150, orient_cost=0.050, height_error=0.050, step_reward=0.450,
                    upper_body_reward=0.050)                                         # tasks/stepping_task.py:107-120
STAND_WEIGHTS = dict(com_vel_error=0.3, yaw_vel_error=0.3, height=0.1, upperbody=0.1, joint_torque_reward=0.1,
                     posture=0.1)                                                    # tasks/standing_task.py:97-104


class _DeviceTask(BaseTask):
    """Common part: the hooks are executed by the step kernel; here they report its results for env `index`."""
    weights: dict = {}

    def __init__(self, env, index: int = 0):
        self._env, self._index = env, index
        self._client = env.interface
        self._control_dt = env.dt
        self._mass = env.mj.get("stepping", {}).get("task_mass", env.mj["total_mass"])      # get_robot_mass()

    def reset(self, iter_count: int = 0) -> None:
        """tasks/*_task.py reset(): runs inside lhw_sim_reset / the auto-reset of lhw_sim_step; the curriculum input travels
        through env.robot.iteration_count."""
        self._env.robot.iteration_count = iter_count

    def step(self) -> None:
        """Runs inside lhw_sim_step (phase advance, mode switches, target tracking)."""

    def calc_reward(self, prev_torque=None, prev_action=None, action=None) -> dict[str, float]:
        terms = self._env.rew_terms[self._index].double().cpu().numpy()
        return {k: float(v) for k, v in zip(self._env.reward_names, terms)}

    def done(self) -> bool:
        return bool(self._env.done[self._index].item())

    # state the reference keeps on the task object, read from the env's integer record [phase mode traj_len ep_len ...]
    @property
    def _phase(self) -> int:
        return int(self._env.state_i[self._index, 0].item())

    @property
    def mode(self) -> int:
        from ..envs.batched_env import MODE_HELD
        return int(self._env.state_i[self._index, 1].item()) & ~MODE_HELD   # without the held-command flag


class WalkingTask(_DeviceTask):
    weights = WALK_WEIGHTS

    def __init__(self, env, index: int = 0):
        super().__init__(env, index)
        cfg = env.mj["cfg"]
        t = cfg["task"]
        self._goal_height_ref, self._total_duration = t["goal_height"], t["total_duration"]
        self._swing_duration, self._stance_duration = t["swing_duration"], t["stance_duration"]
        self._neutral_foot_orient = np.array([1, 0, 0, 0])
        self._period = int(np.floor(2 * self._total_duration * (1 / self._control_dt)))        # tasks/walking_task.py:201
        if env.model_name == "h1_walk":   # the H1 robot: pose in radians (envs/h1/h1_base.py), the bodies StandingTask names
            self._neutral_pose = np.asarray(cfg["half_sitting_pose"], dtype=float)
            self._root_body_name, self._lfoot_body_name, self._rfoot_body_name, self._head_body_name = \
                "pelvis", "left_ankle_link", "right_ankle_link", "torso_link"
        else:
            self._neutral_pose = np.deg2rad(cfg["half_sitting_pose_deg"])
            self._root_body_name, self._lfoot_body_name, self._rfoot_body_name, self._head_body_name = \
                "PELVIS_S", "L_ANKLE_P_S", "R_ANKLE_P_S", "NECK_P_S"                          # envs/jvrc/jvrc_base.py:26-29
        self.manip_hfield = env.model_name == "jvrc_walk_terrain"

    @property
    def mode_ref(self) -> np.ndarray:
        nq, nv, nu = self._env.nq, self._env.nv, self._env.act_dim
        off = nq + 2 * nv + 5 * nu
        return self._env.state_r[self._index, off:off + 3].double().cpu().numpy()


class SteppingTask(WalkingTask):
    weights = STEP_WEIGHTS

    def __init__(self, env, index: int = 0):
        super().__init__(env, index)
        st = env.mj["stepping"]
        self.delay_frames, self.target_radius = st["delay_frames"], st["target_radius"]
        self._lf_site_name, self._rf_site_name = "lf_force", "rf_force"

    @property
    def sequence(self) -> np.ndarray:
        """The footstep sequence [x, y, z, theta] (= the slab poses) of env `index`."""
        s = self._env.state_r[self._index, 119:199].double().cpu().numpy().reshape(20, 4)
        return s[:int(self._env.state_r[self._index, 199].item())]


class StandingTask(_DeviceTask):
    weights = STAND_WEIGHTS

    def __init__(self, env, index: int = 0):
        super().__init__(env, index)
        self._neutral_pose = np.asarray(env.mj["cfg"]["half_sitting_pose"], dtype=float)
        self._root_body_name, self._lfoot_body_name, self._rfoot_body_name, self._head_body_name = \
            "pelvis", "left_ankle_link", "right_ankle_link", "torso_link"


class DeviceRobotInterface:
    """envs/common/robot_interface.py getters answered from the device state record of env `index`; arrays are numpy copies."""

    def __init__(self, env, index: int = 0):
        self._env, self._index = env, index

    def _r(self, lo, n):
        return self._env.state_r[self._index, lo:lo + n].double().cpu().numpy()

    def nq(self): return self._env.nq
    def nv(self): return self._env.nv
    def nu(self): return self._env.act_dim
    def sim_dt(self): return self._env.mj["opt"]["timestep"]
    def get_robot_mass(self): return self._env.mj.get("stepping", {}).get("task_mass", self._env.mj["total_mass"])
    def get_qpos(self): return self._r(0, self._env.nq)
    def get_qvel(self): return self._r(self._env.nq, self._env.nv)
    def get_qacc(self): return self._r(self._env.nq + self._env.nv, self._env.nv)
    def get_gear_ratios(self): return np.ones(self._env.act_dim)                       # gear 1 for both robots

    def get_act_joint_positions(self):          # actuator_length / gear, one substep behind qpos (SURVEY F9)
        return self._r(self._env.nq + 2 * self._env.nv, self._env.act_dim)

    def get_act_joint_velocities(self):
        return self._r(self._env.nq + 2 * self._env.nv + self._env.act_dim, self._env.act_dim)

    def get_act_joint_torques(self):            # actuator_force * gear of the last substep (= prev_torque of the next step)
        return self._r(self._env.nq + 2 * self._env.nv + 4 * self._env.act_dim, self._env.act_dim)

    def get_root_body_pos(self): return self.get_qpos()[0:3]
    def get_root_body_quat(self): return self.get_qpos()[3:7]
    def get_motor_names(self): return [lk["joint"]["name"] for lk in self._env.mj["links"][1:]]


def make_task(env, index: int = 0) -> BaseTask:
    return {"jvrc_walk": WalkingTask, "jvrc_walk_terrain": WalkingTask, "jvrc_step": SteppingTask, "h1": StandingTask,
            "h1_walk": WalkingTask}[env.model_name](env, index)


def model_view(env) -> SimpleNamespace:
    """The few mjModel fields reference code reads off `env.model` (sizes, time step, total mass)."""
    return SimpleNamespace(nq=env.nq, nv=env.nv, nu=env.act_dim, nbody=len(env.mj["links"]) + 1,
                           opt=SimpleNamespace(timestep=env.mj["opt"]["timestep"], gravity=np.array(env.mj["opt"]["gravity"])))


class DataView:
    """`env.data`: qpos / qvel / qacc / time of env `index` as numpy copies of the device record."""

    def __init__(self, env, index: int = 0):
        self._i = DeviceRobotInterface(env, index)

    qpos = property(lambda self: self._i.get_qpos())
    qvel = property(lambda self: self._i.get_qvel())
    qacc = property(lambda self: self._i.get_qacc())
