"""dedalus_b200: H100-native timestep hot loop behind the Dedalus v3 Problem/Solver/Field/basis API.

Public surface mirrors `dedalus.public` (reference dedalus/public.py:4-15) for the Cartesian IVP path.
"""
from .coords import Coordinate, CartesianCoordinates, S2Coordinates, SphericalCoordinates
from .distributor import Distributor
from .basis import (RealFourier, ComplexFourier, Jacobi, Legendre, Ultraspherical,
                    ChebyshevT, ChebyshevU, ChebyshevV, Chebyshev, Fourier)
from .sphere import SphereBasis
from .shell import ShellBasis
from .field import Field
from .operators import (Differentiate, Gradient, Divergence, Laplacian, Trace, TransposeComponents,
                        Interpolate, Integrate, Lift, Convert, TimeDerivative, DotProduct, Multiply, Skew, MulCosine, Curl, curl,
                        grad, div, lap, skew, trace, transpose, integ, ave, dot, interp, Average, UnaryGridFunction,
                        RadialComponent, AngularComponent, radial, angular)
from .problems import IVP, LBVP
InitialValueProblem = IVP
LinearBoundaryValueProblem = LBVP
from .timesteppers import (schemes, CNAB1, SBDF1, CNAB2, MCNAB2, SBDF2, CNLF2, SBDF3, SBDF4,
                           RK111, RK222, RK443, RKSMR, RKGFY)

__version__ = "0.1.0"
from .extras.flow_tools import CFL, GlobalFlowProperty, AdvectiveCFL
