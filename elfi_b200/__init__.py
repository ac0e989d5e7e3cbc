"""elfi_b200 -- H100-native (sm_90a) implementation of ELFI's data-parallel hot path.

The package mirrors the operator / sampler API of elfi-dev/elfi for the batched
summary -> distance -> threshold/top-n selection -> SMC weight path, the BOLFI GP
surrogate, BSL's synthetic likelihood, BOLFIRE's ratio-estimation classifier and the two-stage
summary-statistic selection of Nunes and Balding (TwoStageSelection), robust optimisation Monte
Carlo (ROMC), the local-linear regression adjustment of a sample (adjust_posterior), ABC model
choice between the samples of several models (compare_models) and the Testbench that compares
methods over repeated simulated observations (Rejection repetitions run in lock-step), with the
arithmetic in hand-written CUDA reached through a C ABI (include/elfi_b200.h).
See DESIGN.md and INTEGRATION.md.
"""
__version__ = '0.1.0'

from . import _lib  # noqa: F401
from . import tools  # noqa: F401
from .model import (AdaptiveDistance, Constant, Discrepancy, Distance, ElfiModel,  # noqa: F401
                    NodeReference, Operation, Prior, RandomVariable, Simulator, Summary,
                    get_default_model, new_model, set_default_model)
from .samplers import (SMC, AdaptiveDistanceSMC, AdaptiveThresholdSMC,  # noqa: F401
                       DensityRatioEstimation, GMDistribution, ModelPrior, Rejection)
from .store import OutputPool  # noqa: F401
from .priors import DeviceModelPrior  # noqa: F401
from .bsl import BSL  # noqa: F401
from .bolfire import BOLFIRE, BOLFIREPosterior  # noqa: F401
from .diagnostics import TwoStageSelection  # noqa: F401
from .romc import ROMC  # noqa: F401
from .post_processing import LinearAdjustment, adjust_posterior  # noqa: F401
from .model_selection import compare_models  # noqa: F401
from .testbench import Testbench, TestbenchMethod  # noqa: F401
from .bo import (BOLFI, LCBSC, BayesianOptimization, BolfiPosterior, GPyRegression,  # noqa: F401
                 ExpIntVar, MaxVar, RandMaxVar, UniformAcquisition)
