"""theseus_b200 -- an H100-native (sm_90a) implementation of the batched nonlinear-least-squares inner loop of
facebookresearch/theseus (linearize -> solve -> retract), behind the reference's own plugin API.

    import theseus_b200 as th
    objective = th.Objective(dtype=torch.float64)
    objective.add(th.Between(x0, x1, z, th.DiagonalCostWeight(w)))
    optimizer = th.LevenbergMarquardt(objective.to("cuda"), linear_solver_cls=th.CholeskyDenseSolver, max_iterations=10)
    layer = th.TheseusLayer(optimizer)
    values, info = layer.forward(inputs, optimizer_kwargs=dict(damping=1e-3, adaptive_damping=True, ellipsoidal_damping=True))

All arithmetic runs in libthb200.so (hand-written CUDA behind the C ABI of include/thb200.h); there is no CPU
or PyTorch fallback.  Importing the package does not require a GPU; evaluating anything does.
"""
from .geometry import Variable, Manifold, LieGroup, Vector, Point2, Point3, SE2, SE3, SO2, SO3, as_variable  # noqa: F401
from .core import (AutogradMode, CostWeight, ScaleCostWeight, DiagonalCostWeight, CostFunction, Between, Difference, Local,  # noqa: F401
                   Reprojection, AutoDiffCostFunction, RobustCostFunction, GNCRobustCostFunction, RobustLoss, WelschLoss, HuberLoss,
                   HingeLoss, GNCRobustLoss, GemanMcClureLoss, Objective, masked_jacobians, masked_variables)
from . import embodied as eb  # noqa: F401  (th.eb.Reprojection, like the reference)
from .optimizer import (VariableOrdering, Linearization, DenseLinearization, SparseLinearization, LinearSolver,  # noqa: F401
                        DenseSolver, CholeskyDenseSolver, LUDenseSolver, NonlinearLeastSquares, GaussNewton,
                        LevenbergMarquardt, TrustRegion, Dogleg, NonlinearOptimizerStatus, NonlinearOptimizerInfo, OptimizerInfo,
                        NonlinearOptimizerParams, BackwardMode, convert_to_alpha_beta_damping_tensors, LinearOptimizer, LinearOptimizerStatus, Vectorize)
from .sparse_solver import BaspachoSparseSolver, BlockSparseSolver, CholmodSparseSolver, LUCudaSparseSolver  # noqa: F401
from .layer import TheseusLayer  # noqa: F401
from .functional import (adjoint, between, compose, exp_map, inverse, local, log_map, retract, rand_vector, randn_vector,  # noqa: F401
                         rand_point2, randn_point2, rand_point3, randn_point3, rand_so3, randn_so3, rand_se3, randn_se3, rand_se2, randn_se2,
                         rand_so2, randn_so2)
from . import io_formats  # noqa: F401  (g2o / BAL readers: th.io_formats.read_3D_g2o_file, load_bal_dataset)

from .geometry import enable_lie_group_check, no_lie_group_check, set_lie_group_check_enabled  # noqa: F401,E402

from . import geometry_api as _geometry_api  # noqa: E402
_geometry_api.install()

__version__ = "0.1.0"
