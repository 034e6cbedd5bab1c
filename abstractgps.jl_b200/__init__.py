"""agp-blackwell: H100-native exact-GP engine behind AbstractGPs.jl's public surface.

`from agp_b200 import *` gives the reference's names (GP, FiniteGP via f(x, s2), logpdf, posterior,
mean_and_var, rand, VFE, elbo, kernels and transforms).  All arithmetic runs in libagp.so
(hand-written sm_90a CUDA, C ABI in include/agp.h); importing this package does not need a GPU,
calling into it does -- there is no CPU fallback."""
from .api import *  # noqa: F401,F403
from .api import (AGPError, DimensionMismatch, PosDefException, engine, Engine, fit, rand_from_normals,
                  Xt_invA_X, Xt_invA_Y, diag_Xt_invA_X, tr_Xt_invA_X, DeviceCholesky, vcat)
from . import _cabi  # noqa: F401

__version__ = "0.1.0"
