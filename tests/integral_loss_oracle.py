"""Float64 restatement of an integral constraint as additional loss (pinn.IntegralLoss): oracle.reference's Problem with
``full_loss`` = Σ_k w_k L_k + w_add · g(Σ_p w_p v_p - target), g = |·| or (·)², v_p the integrand at node p
(src/discretize.jl:590-597 adds additional_loss after the weighted sum), and its gradient by torch autograd.  The
integrand is evaluated like an equation side, with exact derivatives (the engine's forward-mode taps)."""
import numpy as np
import sympy as sp
import torch

from neuralpde_jl_b200.symbolic import Equation
from oracle import reference as R


class IntegralLossProblem(R.Problem):
    """R.Problem with one integral constraint.  X: (d, n) nodes (rows = the integrand's variables in eq_indvars
    order), w: (n,) weights."""

    def __init__(self, *args, integrand, X, w, target: float = 0.0, norm: str = "abs", w_add: float = 1.0, **kw):
        kw.setdefault("derivative", "exact")
        super().__init__(*args, **kw)
        self.eq_f = Equation(sp.sympify(integrand), sp.Integer(0))
        self.X = torch.as_tensor(np.asarray(X, dtype=np.float64))
        self.w = torch.as_tensor(np.asarray(w, dtype=np.float64))
        self.target, self.norm, self.w_add = float(target), norm, float(w_add)

    def values(self, theta) -> torch.Tensor:
        """v_p at every node"""
        return self.residual(self.eq_f, self.X, theta)[0]

    def functional(self, theta) -> torch.Tensor:
        s = torch.sum(self.w * self.values(theta)) - self.target
        return torch.abs(s) if self.norm == "abs" else s * s      # torch's |·|' at 0 is 0, as Zygote's sign(0)

    def loss_and_grad(self, theta_np, pde_sets, bc_sets, **kw):
        return super().loss_and_grad(theta_np, pde_sets, bc_sets, extra=(self.w_add, self.functional), **kw)
