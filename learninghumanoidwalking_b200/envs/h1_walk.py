"""H1WalkEnv — single-environment view of the Unitree H1 walking environment: the H1 robot of H1Env (observation noise,
per-episode dynamics randomisation, random pushes, initial-pose noise) with the WalkingTask of JvrcWalkEnv (gait clock, mode
machine, 10 reward terms).  A 1-env BatchedHumanoidEnv(model="h1_walk"); which constants this build defines is in DESIGN.md §4.6."""
from __future__ import annotations

from .jvrc_walk import JvrcWalkEnv


class H1WalkEnv(JvrcWalkEnv):
    MODEL = "h1_walk"
