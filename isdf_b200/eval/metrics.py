"""Mirror of reference isdf/eval/metrics.py: step timing (metrics.py:13-38, milliseconds, CUDA events on GPU) and the
collision costs (metrics.py:95-113).  The other functions of that module are not provided here."""
import time

import torch


def start_timing():
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        start = torch.cuda.Event(enable_timing=True)
        end = torch.cuda.Event(enable_timing=True)
        start.record()
        return start, end
    return time.perf_counter(), None


def end_timing(start, end):
    if torch.cuda.is_available():
        end.record()
        end.synchronize()
        return start.elapsed_time(end)
    return (time.perf_counter() - start) * 1000.0


def chomp_cost(sdf, epsilon=2.0):
    """CHOMP collision cost (Zucker et al., IJRR 2013, eq. 21) of each SDF value of a numpy array or torch tensor:
    -s + epsilon / 2 for s <= 0, (s - epsilon)^2 / (2 epsilon) for 0 < s <= epsilon, 0 above epsilon; NaN stays NaN.
    Returns a new array of the input's kind and dtype, filled in place branch by branch in the reference's arithmetic
    (the quadratic as 1 / (2 epsilon) times the square)."""
    cost = -sdf + epsilon / 2.
    near = sdf > 0
    cost[near] = 1 / (2 * epsilon) * (sdf[near] - epsilon) ** 2
    cost[sdf > epsilon] = 0.
    return cost


def linear_cost(sdf, epsilon=1.5):
    """Linear collision cost of each SDF value: epsilon - s up to epsilon, 0 above it; a new array as chomp_cost."""
    cost = -sdf + epsilon
    cost[sdf > epsilon] = 0.
    return cost
