"""A minimal stand-in for the three pyunlocbox names pygsp/learning.py:42-180
(classification_tikhonov_simplex) uses, so that the reference's own function -- its
``proj_simplex``, ``smooth_eval`` and ``smooth_grad`` included -- runs unchanged without the
package.  This is NOT pyunlocbox.  It restates only the behaviour that function relies on:

* ``functions.func``: an object whose ``_eval`` / ``_grad`` / ``_prox`` attributes the caller
  sets; ``eval(x)``, ``grad(x)`` and ``prox(x, T)`` call them.
* ``solvers.forward_backward(step=...)`` with FISTA acceleration: ``t = 1`` at the first
  iteration; at every iteration ``t' = (1 + sqrt(1 + 4 t^2)) / 2``,
  ``y = x_k + ((t - 1) / t') (x_k - x_{k-1})``, ``t = t'``, then
  ``x_{k+1} = prox(y - step grad(y), step)`` of the second function, the first being the smooth
  one.
* ``solvers.solve(functions, x0, solver, atol=None, dtol=None, rtol=1e-3, xtol=None, maxit=200,
  verbosity='LOW')``: the objective (the sum of the functions' ``eval``) is taken at x0 and at
  every new iterate; after iteration k the tests, in this order, each overriding the previous
  one, are ``cur < atol`` -> 'ATOL', ``|cur - last| < dtol`` -> 'DTOL',
  ``|cur - last| / |cur| < rtol`` -> 'RTOL' (divided by ``last`` when ``cur == 0``, ratio 0 when
  both are 0), ``||x_k - x_{k-1}|| / sqrt(x.size) < xtol`` -> 'XTOL' and ``k >= maxit`` ->
  'MAXIT'.  It returns ``{'sol', 'crit', 'niter', 'objective'}`` (objective: one
  ``[f1, f2]`` list per evaluation).  ``verbosity`` is accepted and ignored.

``install()`` puts the modules into ``sys.modules`` as ``pyunlocbox``, ``pyunlocbox.functions``
and ``pyunlocbox.solvers``.
"""
import sys
import types

import numpy as np


class func:
    def eval(self, x):
        return self._eval(x)

    def grad(self, x):
        return self._grad(x)

    def prox(self, x, T):
        return self._prox(x, T)


class forward_backward:
    def __init__(self, step=1.0):
        if step <= 0:
            raise ValueError("Step should be a positive number.")
        self.step = step

    def pre(self, functions, x0):
        if len(functions) != 2:
            raise ValueError("forward_backward requires two convex functions.")
        self.smooth, self.non_smooth = functions
        self.sol = np.array(x0, copy=True, dtype=np.float64)
        self.prev = np.array(x0, copy=True, dtype=np.float64)
        self.t = 1.0

    def algo(self, niter):
        if niter == 1:
            self.t = 1.0
        t = (1.0 + np.sqrt(1.0 + 4.0 * self.t ** 2.0)) / 2.0
        y = self.sol + ((self.t - 1) / t) * (self.sol - self.prev)
        self.t = t
        self.prev[:] = self.sol
        x = y - self.step * self.smooth.grad(y)
        self.sol[:] = self.non_smooth.prox(x, self.step)


def solve(functions, x0, solver, atol=None, dtol=None, rtol=1e-3, xtol=None, maxit=200,
          verbosity="LOW"):
    if verbosity not in ("NONE", "LOW", "HIGH", "ALL"):
        raise ValueError("Verbosity should be either NONE, LOW, HIGH or ALL.")
    crit, niter = None, 0
    objective = [[f.eval(x0) for f in functions]]
    solver.pre(functions, x0)
    while not crit:
        niter += 1
        last_sol = np.array(solver.sol, copy=True)
        solver.algo(niter)
        objective.append([f.eval(solver.sol) for f in functions])
        current, last = np.sum(objective[-1]), np.sum(objective[-2])
        if atol is not None and current < atol:
            crit = "ATOL"
        if dtol is not None and np.abs(current - last) < dtol:
            crit = "DTOL"
        if rtol is not None:
            div = current
            if div == 0:
                div = last if last != 0 else 1.0
            if np.abs((current - last) / div) < rtol:
                crit = "RTOL"
        if xtol is not None:
            err = np.linalg.norm(solver.sol - last_sol) / np.sqrt(last_sol.size)
            if err < xtol:
                crit = "XTOL"
        if maxit is not None and niter >= maxit:
            crit = "MAXIT"
    return {"sol": solver.sol, "crit": crit, "niter": niter, "objective": objective}


def install():
    """Register the stand-in as ``pyunlocbox`` (returns the package module)."""
    pkg = types.ModuleType("pyunlocbox")
    functions = types.ModuleType("pyunlocbox.functions")
    solvers = types.ModuleType("pyunlocbox.solvers")
    functions.func = func
    solvers.forward_backward = forward_backward
    solvers.solve = solve
    pkg.functions, pkg.solvers = functions, solvers
    pkg.__doc__ = "stand-in (oracle/unlocbox_standin.py), not pyunlocbox"
    sys.modules.update({"pyunlocbox": pkg, "pyunlocbox.functions": functions,
                        "pyunlocbox.solvers": solvers})
    return pkg
