"""oracle/ for h1_walk (tests only): the H1 robot with the WalkingTask, composed from what oracle/sim_oracle.c already computes.

The oracle's physics, randomisation, pushes, initial-pose noise, gait clock, mode machine, rewards and termination are all driven
by the packed model, so h1.json's robot with a WalkingTask tail (task 0) and h1's noise / randomisation values runs there as it
is.  Only the observation is the standing task's robot state plus the walking task's words, which the oracle's WalkingTask does
not assemble: `observe` builds the 43 words from the oracle's 33 (roll, pitch, angular velocity, joint positions and velocities,
then the 8 walking words), its motor torques (`act_force`) and the uniform observation noise of h1 on the 35 robot-state words,
drawn as sim_oracle.c get_obs draws it for h1: value i -> Philox stream 40 + i/4, lane i%4, at the env's event counter."""
import ctypes

import numpy as np

from oracle import oracle as O

NU, NROBOT, NOBS = 10, 35, 43
TORQUES = slice(25, 35)


def pack_oracle_model(mj: dict, clocks: dict, tolerance=None) -> np.ndarray:
    """oracle.pack_model's WalkingTask layout for the H1 model, with h1's noise / randomisation tail in place of the zeros."""
    t = mj["cfg"]["task"]
    assert (clocks["swing"], clocks["stance"]) == (t["swing_duration"], t["stance_duration"]), "the golden clock table is jvrc_walk's"
    flat = O.pack_model(mj, clocks, tolerance)
    # words after the task tail: per geom (type, npts, radius, points), root parts (29), pdrand_k, terrain flag, assumption flags
    after = sum(3 + 3 * len(g.get("points", [])) for g in mj["geoms"]) + 29 + 3
    k = len(flat) - after - 14
    assert list(flat[k:k + 4]) == [0, 37, 0.6, 1.4], flat[k:k + 4]
    c = mj["cfg"]
    ns, pert, dyn = c["observation_noise"], c["perturbation"], c["dynamics_randomization"]
    lvl = ns["multiplier"] if ns["enabled"] else 0.0
    flat[k:k + 14] = [0, NOBS - NU, 0.6, 1.4] + [lvl * ns["scales"][s] for s in ("root_orient", "root_ang_vel", "motor_pos",
                                                                                 "motor_vel", "motor_tau")] + \
        [int(dyn["interval"] / c["control_dt"]) if dyn["enable"] else 0, int(pert["interval"] / c["control_dt"]) if pert["enable"] else 0,
         pert["force_magnitude"], pert["torque_magnitude"], c["init_noise_deg"]]
    return flat


class H1WalkOracle(O.Oracle):
    def __init__(self, tolerance=None):
        self.lib = ctypes.CDLL(O.build())
        L = self.lib
        L.orc_energy.restype = ctypes.c_double
        self.mj, self.clocks = O.load_model_json("h1_walk"), O.load_clocks()
        flat = pack_oracle_model(self.mj, self.clocks, tolerance)
        self._model = ctypes.create_string_buffer(L.orc_sizeof_model())
        rc = L.orc_model_from_flat(self._model, flat.ctypes.data_as(ctypes.c_void_p), len(flat))
        if rc != 0:
            raise RuntimeError(f"orc_model_from_flat failed: {rc}")
        self.env_size = L.orc_sizeof_env()
        self.nu, self.nv, self.nq = NU, 6 + NU, 7 + NU
        self.nobs = NOBS - NU          # what the oracle's WalkingTask writes
        k = len(flat) - sum(3 + 3 * len(g.get("points", [])) for g in self.mj["geoms"]) - 29 - 3 - 14
        s = flat[k + 4:k + 9]
        self.noise = np.array([s[0]] * 2 + [s[1]] * 3 + [s[2]] * NU + [s[3]] * NU + [s[4]] * NU)

    def observe(self, envs, obs33, back=None):
        """The 43-word observation of every env from the oracle's 33 words.  `back` (per env, 0 / 1): the draw is that many event
        counters back (a terminal observation whose env has since been reset); its torque words are then unknown (NaN)."""
        n = obs33.shape[0]
        back = np.zeros(n, int) if back is None else np.asarray(back, int)
        out = np.empty((n, NOBS))
        for i in range(n):
            tq = self.field(envs, i, "act_force")[:NU] if not back[i] else np.full(NU, np.nan)
            robot = np.concatenate((obs33[i, :25], tq))
            seed, env_id = int(self.field(envs, i, "seed")[0]), int(self.field(envs, i, "env_id")[0])
            ctr = int(self.field(envs, i, "rng_ctr")[0]) - back[i]
            for j in range(NROBOT):
                sc = float(self.noise[j])
                if sc > 0:
                    u = self.philox(seed, env_id, ctr, 40 + (j >> 2))[j & 3]
                    robot[j] += -sc + 2 * sc * ((u >> 8) * (1.0 / 16777216.0))
            out[i] = np.concatenate((robot, obs33[i, 25:]))
        return out

    def batch_reset(self, envs, n, nthreads=0):
        return self.observe(envs, super().batch_reset(envs, n, nthreads))

    def batch_step(self, envs, n, actions, max_traj_len=400, nthreads=0):
        obs, tobs, terms, rew, done, ended = super().batch_step(envs, n, actions, max_traj_len, nthreads)
        return self.observe(envs, obs), self.observe(envs, tobs, back=ended), terms, rew, done, ended
