from .ddim import DDIMScheduler  # noqa: F401
from .ddpm import DDPMScheduler  # noqa: F401
from .dpm_solver import DPMSolverMultistepScheduler  # noqa: F401
from .pndm import PNDMScheduler  # noqa: F401
from .sa_solver import SASolverScheduler  # noqa: F401
from .scheduler import NoiseSchedules, Scheduler  # noqa: F401
from .unipc import UniPCMultistepScheduler  # noqa: F401
