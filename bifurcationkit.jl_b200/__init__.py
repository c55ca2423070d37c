"""bk200: H100-native Newton-Krylov corrector for BifurcationKit-style pseudo-arclength
continuation.  The directory name carries a dot (bifurcationkit.jl_b200), so import it through
``__graft_entry__.load_package()`` (registers it as the module ``bk200``).

Contents: csrc/ (CUDA kernels + C ABI -> libbk200.so), lib.py (ctypes binding), core.py (mirror of
the reference's AbstractLinearSolver / AbstractBorderedLinearSolver / AbstractEigenSolver surfaces),
palc.py (host-side Newton / newton_palc / continuation loop driving the device kernels), defcont.py (deflated
continuation), periodic.py (periodic-orbit
branches with the Trapeze functional and branch switching to them from a Hopf point), bifdiagram.py (automatic bifurcation
diagrams, sibling branches continued concurrently).
"""
from . import lib
from .lib import (BK200Error, BK_CHAN, BK_SH2D, BK_SH3D, BK_CGL2D, BK_POTRAP_CGL2D, BK_SH2D_PERIODIC, BK_RD, BK_COMPLEX, BK_PC_NONE,
                  BK_PC_SH_DCT, BK_PC_CHAN_TRIDIAG, BK_PC_CGL_DST, BK_PC_POTRAP_CIRC, BK_PC_SH_FFT, BK_PC_RD, BK_BC_NEUMANN,
                  BK_BC_DIRICHLET, build)
from .core import (Context, ReactionDiffusion, DeviceVec, Jacobian, TransposedJacobian, ComplexJacobian, GMRESB200, ComplexGMRESB200, BorderingBLSB200, MatrixFreeBLSB200, ShiftInvertB200,
                   bls_map, bls_map_block, make_opts, hessenberg_eig)
from . import palc
from . import segments
from . import floquet
from . import events
from . import deflation
from . import defcont
from . import codim2
from . import normalform
from . import periodic
from . import bifdiagram
