"""iterativesolvers.jl_b200 -- host-side mirror of IterativeSolvers.jl's hot-path interface over the
B200-native C ABI (libb200krylov.so).

Julia is not available in this image, so this Python layer plays the role of the Julia shim
(INTEGRATION.md): same function names (`cg!` -> `cg_`), keyword arguments, defaults, return shapes
(`x` or `(x, ConvergenceHistory)`) and error behaviour as reference src/cg.jl, src/gmres.jl,
src/minres.jl, src/bicgstabl.jl, src/lobpcg.jl (and, as the section 8(f) widening, src/chebyshev.jl, src/qmr.jl,
src/lsqr.jl, src/lsmr.jl, src/idrs.jl).  All arithmetic runs in the CUDA library; this
package contains no numerical fallback.

The directory name contains a dot, so import it through the repo-root alias module:
    import iterativesolvers_jl_b200 as isb
"""
from ._lib import B200Error, lib  # noqa: F401
from .device import Context, DeviceArray, default_context, pinned_empty  # noqa: F401
from .operators import (B200CSR, B200LinearOperator, FunctionPrec, HaloPlan, Identity, ILU0Prec, JacobiPrec,  # noqa: F401
                        SmoothedAggregationPrec, aspreconditioner, smoothed_aggregation)
from .history import ConvergenceHistory, niters, nprods, nrests  # noqa: F401
from .generators import laplace_matrix, laplace_csr_slab, advection_dominated, mmread, matread  # noqa: F401
from .solvers import (cg, cg_, chebyshev, chebyshev_, gmres, gmres_, minres, minres_, bicgstabl, bicgstabl_, lobpcg,  # noqa: F401
                      LOBPCGResults, orthogonalize_and_normalize_, hessenberg_ldiv_,
                      cg_iterator_, CGIterable, CGStateVariables, KrylovIterable, gmres_iterable_, minres_iterable_,
                      bicgstabl_iterator_, minres_iterable, bicgstabl_iterator, LOBPCGIterator, lobpcg_, powm_, powm, invpowm_, invpowm, jacobi_, jacobi, gauss_seidel_, gauss_seidel,
                      sor_, sor, ssor_, ssor,
                      qmr, qmr_, lsqr, lsqr_, lsmr, lsmr_, idrs, idrs_, LobpcgConstraint, svdl, SVD,
                      PartialFactorization)

# type names the reference exports for its iterables (src/cg.jl:3, src/bicgstabl.jl:3): one device class serves both CG
# variants (the preconditioner decides), and the fused-pass iterables share a class
PCGIterable = CGIterable
BiCGStabIterable = KrylovIterable
