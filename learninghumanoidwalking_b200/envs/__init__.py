from .batched_env import BatchedHumanoidEnv  # noqa: F401
from .h1 import H1Env  # noqa: F401
from .h1_walk import H1WalkEnv  # noqa: F401
from .jvrc_walk import JvrcWalkEnv  # noqa: F401
from .jvrc_step import JvrcStepEnv  # noqa: F401
