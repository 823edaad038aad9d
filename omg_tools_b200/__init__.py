"""omg_tools_b200: CUDA-native batched solver for OMG-tools' per-MPC-step
spline-trajectory NLP, behind the reference's Problem.solve()/OptiFather API."""
from .basics.spline import BSplineBasis, BSpline
from .basics.shape import (Circle, Polyhedron, Rectangle, Square, Beam,
                           RegularPolyhedron, Sphere, Cuboid, Cube, Plate,
                           RegularPrisma)
from .basics.optilayer import OptiChild, OptiFather, create_nlp
from .vehicles.vehicle import Vehicle
from .vehicles.holonomic import Holonomic
from .vehicles.holonomic3d import Holonomic3D
from .vehicles.holonomic1d import Holonomic1D
from .vehicles.holonomicorient import HolonomicOrient
from .vehicles.quadrotor import Quadrotor
from .vehicles.dubins import Dubins
from .vehicles.bicycle import Bicycle
from .vehicles.agv import AGV
from .vehicles.trailer import Trailer
from .vehicles.quadrotor3d import Quadrotor3D
from .vehicles.quadrotor3d_simple import SimpleQuadrotor3D
from .vehicles.fleet import Fleet
from .environment.environment import Environment
from .environment.obstacle import Obstacle
from .problems.problem import Problem
from .problems.point2point import Point2point, FixedTPoint2point, FreeEndPoint2point
from .problems.formation_central import FormationPoint2pointCentral
from .problems.admm import FormationPoint2point, RendezVous

__version__ = '0.1.0'
