"""neuralpde.jl_b200 -- H100-native PINN residual/loss engine behind NeuralPDE.jl's
PhysicsInformedNN / discretize interface.

The directory name contains a dot, so import it through the root-level alias module:
``import neuralpde_jl_b200 as npde``.
"""
from .engine import (Engine, EngineError, FixedNetSpec, IntegralSpec, NetSpec, ProblemSpec, TapSpec, TermSpec, EXPORTS, LIB_PATH,
                     MODE_FFMA, MODE_TC_BF16, MODE_TC_SPLIT, MODE_TC_F64, REDUCE_ABS_OF_SUM, REDUCE_MEAN, REDUCE_SQUARE_OF_SUM,
                     REDUCE_WSUM, load_library)
from .symbolic import (ClosedInterval, Differential, Eq, Equation, In, Inf, Integral, Interval, PDESystem,
                       ProductDomain, UnitInterval, UnitSquare, VarDomain, get_argument, get_variables, get_vars,
                       parameters, variables)
from .lowering import LoweringError, lower_equation
from .strategies import (AbstractTrainingStrategy, GridTraining, QuadratureTraining, QuasiRandomTraining,
                         StochasticTraining, WeightedIntervalTraining, generate_training_sets, get_bounds, shard_range)
from .pinn import (AbstractPINN, Adam, BPINNsolution, BPINNstats, DiagEuclideanMetric, HMC, Leapfrog, LogNormal,
                   NoAdaptation, Normal, Uniform,
                   StanHMCAdaptor, UnitEuclideanMetric, ahmc_bayesian_pinn_pde, pmean, BFGS, BackTracking, BayesianPINN, Chain, DataLoss, Dense, IntegralLoss, Descent, GradientScaleAdaptiveLoss, HagerZhang, LBFGS, LogOptions, MiniMaxAdaptiveLoss,
                   NonAdaptiveLoss, ReLoBRaLoAdaptiveLoss, SoftAdaptAdaptiveLoss,
                   OptimizationFunction, OptimizationProblem, Phi, PhysicsInformedNN, PINNRepresentation, Solution,
                   discretize, initialparameters, logscalar, logvector, register_symbolic, solve, symbolic_discretize)
from .adapter import NeuralAdapterLoss, neural_adapter
from .ode import NNODE, NNODERepresentation, ODEFunction, ODEProblem, ODESolution
from .bpinn_ode import BNNODE, BNNODELogDensity, ahmc_bayesian_pinn_ode
from .sde import NNSDE, NNSDERepresentation, SDEProblem, SDEsol
from .sde_weak import SDEPINN
from .dae import DAEFunction, DAEProblem, DAESolution, NNDAE, NNDAERepresentation

__all__ = [n for n in dir() if not n.startswith("_")]
