"""Float64 restatement of the reference's Bayesian ODE log density ``LogTargetDensity``
(ext/bpinn/advancedHMC_MCMC.jl:43-254), term by term with Gaussian logpdfs, on top of tests/nnode_oracle.py's trial
solution and f.  Independent of bpinn_ode.py's term table: the physics times of every evaluation are passed in."""
import math

import numpy as np
import torch

from nnode_oracle import NNODEOracle

LOG2PI = math.log(2.0 * math.pi)


def normal_logpdf_sum(x, mean, std):
    """Σ_i logpdf(Normal(mean_i, std), x_i): MvNormal(mean, std² I) at x"""
    n = x.numel()
    return -((x - mean) ** 2).sum() / (2.0 * std * std) - 0.5 * n * LOG2PI - n * torch.log(torch.abs(torch.as_tensor(std)))


def prior_logpdf(kind, a, b, x):
    if kind == "normal":
        return -((x - a) / b) ** 2 / 2 - 0.5 * LOG2PI - math.log(b)
    if kind == "lognormal":
        lx = torch.log(x)
        return -((lx - a) / b) ** 2 / 2 - 0.5 * LOG2PI - math.log(b) - lx
    return torch.as_tensor(-math.log(b - a), dtype=torch.float64)


class BNNODEOracle:
    """``phynewstd(p_list) -> list`` is called with θ.p as a list of torch scalars (inverse) or the problem's p."""

    def __init__(self, prob, chain, *, param=(), dataset=(), phystd=(0.05,), l2std=(0.05,), phynewstd=None,
                 estim_collocate=False, priorsNNw=(0.0, 2.0), derivative="exact"):
        self.o = NNODEOracle(prob, chain, param_estim=len(param) > 0)
        self.param = list(param)          # [(kind, a, b)] in θ.p order
        self.dataset = [np.asarray(v, dtype=np.float64) for v in dataset]
        self.phystd, self.l2std = list(phystd), list(l2std)
        self.phynewstd, self.estim_collocate = phynewstd, estim_collocate
        self.priorsNNw, self.derivative = priorsNNw, derivative
        self.n, self.n_net = self.o.n, self.o.n_net

    def physloglikelihood(self, th, times=None, quad=None):
        """times: per component, the times of its MvNormal (the dataset's appended); quad: (nodes, weights) for
        QuadratureTraining (∫ of innerdiff's one-point logpdf)"""
        out = torch.zeros((), dtype=torch.float64)
        if quad is not None:
            x = torch.tensor(quad[0], dtype=torch.float64)
            w = torch.tensor(quad[1], dtype=torch.float64)
            r = self.o.residual(th, x, self.derivative)
            for k in range(self.n):
                s = self.phystd[k]
                out = out + (w * (-r[k] ** 2 / (2 * s * s) - 0.5 * LOG2PI - math.log(s))).sum()
            return out
        for k in range(self.n):
            t = torch.tensor(np.asarray(times[k], dtype=np.float64))
            r = self.o.residual(th, t, self.derivative)
            out = out + normal_logpdf_sum(torch.zeros_like(t), r[k], self.phystd[k])
        return out

    def priorweights(self, th):
        mu, sd = self.priorsNNw
        net = th[:self.n_net]
        out = normal_logpdf_sum(net, torch.full_like(net, float(mu)), float(sd))
        for j, (kind, a, b) in enumerate(self.param):
            out = out + prior_logpdf(kind, a, b, th[self.n_net + j])
        return out

    def l2lossdata(self, th):
        if not self.dataset:
            return torch.zeros((), dtype=torch.float64)
        t = torch.tensor(self.dataset[-2])
        ph = self.o.phi(th, t)
        return sum(normal_logpdf_sum(torch.tensor(self.dataset[k]), ph[k], self.l2std[k]) for k in range(self.n))

    def l2loss2(self, th):
        if not self.estim_collocate:
            return torch.zeros((), dtype=torch.float64)
        t = torch.tensor(self.dataset[-2])
        W = torch.tensor(self.dataset[-1])
        uh = torch.stack([torch.tensor(self.dataset[j]) for j in range(self.n)])
        d = self.o.dphi(th, t, self.derivative) - self.o.fval(uh, th, t)
        p = self.o.p_of(th)
        sig = self.phynewstd(p[0] if np.ndim(self.o.prob.p) == 0 and p else p)
        return sum(normal_logpdf_sum(torch.zeros_like(t), d[k] * W, sig[k]) for k in range(self.n))

    def loglik(self, th, times=None, quad=None):
        """the log density without priorweights"""
        return self.physloglikelihood(th, times, quad) + self.l2lossdata(th) + self.l2loss2(th)

    def logdensity(self, th, times=None, quad=None):
        return self.loglik(th, times, quad) + self.priorweights(th)

    def value_grad(self, theta, fn):
        th = torch.tensor(np.asarray(theta, dtype=np.float64), requires_grad=True)
        v = fn(th)
        (g,) = torch.autograd.grad(v, th)
        return float(v.detach()), g.numpy()
