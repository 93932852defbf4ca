"""H100-native batched minimum-derivative trajectory solve (drop-in for
mav_trajectory_generation::PolynomialOptimization<N>::solveLinear()).

Python here is plumbing for tests and benchmarks; the product is the C-ABI library
(include/mtg_b200.h, csrc/) and the C++ host mirror (host/)."""
from . import _build  # noqa: F401
from .capi import (KERNEL_GENERIC, KERNEL_NOFREE, KERNEL_WAYPOINT, STATUS_BAD_TIME,  # noqa: F401
                   STATUS_NOT_SPD, TIME_COST_RICHTER, TIME_COST_SQUARED, Problem, Solver, load,
                   time_objective_params, mellinger_params)
