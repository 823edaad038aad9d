"""BASELINE.json scenario builders (SURVEY.md section 8d), shared by tests and
bench.py.  Each returns an initialised problem whose ``father.tables`` is the
lowered structure; instance data (x0, p) come from ``instance_data``."""
import numpy as np

from . import (Holonomic, Environment, Obstacle, Point2point, Square, Circle,
               Beam, Rectangle)


def _p2p(vehicle, environment, options, build_solver, freeT=False):
    opts = {'verbose': 0}
    opts.update(options or {})
    problem = Point2point(vehicle, environment, options=opts, freeT=freeT)
    if build_solver:
        problem.init()
    else:
        # model + tables only (no CUDA library needed): used by the CPU tests
        problem.father.reset()
        problem.construct()
        f = problem.father
        f.translate_symbols()
        f.construct_variables()
        f.construct_parameters()
        rows, lb, ub = f.construct_constraints()
        from .basics.lowering import lower
        f.tables = lower(f._var_ids, f._par_ids, rows, f.construct_objective(),
                         lb, ub, f.order_hint())
        f.init_variables()
        f.init_parameters()
        f.init_transformations(problem.init_primal_transform,
                               problem.init_dual_transform)
    problem.reinitialize()
    return problem


def config1(options=None, build_solver=True):
    """examples/p2p_holonomic.py as written at the surveyed commit: one moving
    Circle(0.5) obstacle, safety_distance 0.1 (n=98, m=325, n_par=17)."""
    vehicle = Holonomic()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    trajectories = {'velocity': {'time': [0., 40.],
                                 'values': [[-0.35, 0.35], [0., 0.15]]}}
    environment.add_obstacle(Obstacle(
        {'position': [1.5, -1]}, shape=Circle(0.5), options={'bounce': False},
        simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver)


CONFIG2_OBSTACLES = [(-0.5, -0.3), (0.6, 0.4), (1.4, -0.6)]


def config2(options=None, build_solver=True):
    """batch Holonomic Point2point, 3 static Circle(0.4) obstacles, sd=0.1
    (n=190, m=563, n_par=35); layout fixed by SURVEY.md section 8d."""
    vehicle = Holonomic()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    for pos in CONFIG2_OBSTACLES:
        environment.add_obstacle(Obstacle({'position': list(pos)},
                                          shape=Circle(0.4)))
    return _p2p(vehicle, environment, options, build_solver)


def config5(options=None, build_solver=True):
    """examples/revolving_door.py: 2 static + 2 rotating Beam obstacles
    (n=184, m=862)."""
    vehicle = Holonomic()
    vehicle.set_initial_conditions([0., -2.0])
    vehicle.set_terminal_conditions([0., 2.0])
    environment = Environment(room={'shape': Square(5.)})
    beam1 = Beam(width=2.2, height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2., 0.]}, shape=beam1))
    environment.add_obstacle(Obstacle({'position': [2., 0.]}, shape=beam1))
    beam2 = Beam(width=1.4, height=0.2)
    horizon_time = 10.
    omega = 1.5 * (2 * np.pi / horizon_time)
    environment.add_obstacle(Obstacle(
        {'position': [0., 0.], 'velocity': [0., 0.], 'angular_velocity': omega},
        shape=beam2, simulation={}, options={'horizon_time': horizon_time}))
    environment.add_obstacle(Obstacle(
        {'position': [0., 0.], 'velocity': [0., 0.], 'orientation': 0.5 * np.pi,
         'angular_velocity': omega},
        shape=beam2, simulation={}, options={'horizon_time': horizon_time}))
    opts = {'horizon_time': horizon_time}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def config_holonomic3d(options=None, build_solver=True, start=(-2., -2., -2.),
                        goal=(2., 2., -2.)):
    """examples/p2p_holonomic_3d.py: Plate vehicle in a Cube(5) room, a static
    Cuboid and a rising RegularPrisma obstacle, hard terminal constraints,
    horizon 12 s (n=166, m=1536, n_par=109)."""
    from . import Holonomic3D, Plate, Cube, Cuboid, RegularPrisma
    vehicle = Holonomic3D(Plate(Rectangle(0.5, 1.), height=0.1))
    # NB the example's start and goal put the plate exactly on the room limit:
    # jittered copies need interior points
    vehicle.set_initial_conditions(list(start))
    vehicle.set_terminal_conditions(list(goal))
    environment = Environment(room={'shape': Cube(5.)})
    environment.add_obstacle(Obstacle(
        {'position': [0., 0., -1.5]}, shape=Cuboid(width=0.5, depth=4., height=2.)))
    trajectories = {'velocity': {'time': [4.], 'values': [[0.0, 0.0, 1.]]}}
    environment.add_obstacle(Obstacle(
        {'position': [1., 1., -2.25]}, shape=RegularPrisma(0.25, 0.25, 6),
        simulation={'trajectories': trajectories}))
    opts = {'hard_term_con': True, 'horizon_time': 12}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def config4(n_obstacles=2, options=None, build_solver=True):
    """examples/p2p_3dquadrotor.py: Quadrotor3D(0.5), Cuboid(8,6,8) room,
    safety distance 0.1 / weight 10, horizon 5 s, knot_intervals 10
    (SURVEY.md section 8d: 13 is not usable in the reference).  n_obstacles=2
    is the example (two upright plates, the second sinking; n=238, m=1319);
    n_obstacles=5 adds three more static plates (BASELINE config 4, n=406)."""
    from . import Quadrotor3D, Plate, Cuboid
    vehicle = Quadrotor3D(0.5)
    vehicle.set_initial_conditions([-3, -2, -0.5, 0, 0, 0, 0, 0])
    vehicle.set_terminal_conditions([3, 2, 0.5])
    vehicle.set_options({'safety_distance': 0.1, 'safety_weight': 10})
    environment = Environment(room={'shape': Cuboid(8, 6, 8)})
    plate = lambda: Plate(Rectangle(5., 8.), 0.1, orientation=[0., np.pi / 2, 0.])
    trajectory = {'velocity': {'time': [1.5], 'values': [[0, 0, -0.6]]}}
    environment.add_obstacle(Obstacle({'position': [-2, 0, -2]}, shape=plate()))
    environment.add_obstacle(Obstacle({'position': [2, 0, 3.5]}, shape=plate(),
                                      simulation={'trajectories': trajectory}))
    extra = [([0., 0., -3.5], Plate(Rectangle(1., 8.), 0.1, orientation=[0., np.pi / 2, 0.])),
             ([-3.5, 2.5, 3.], Plate(Rectangle(1., 1.), 0.1)),
             ([3.5, -2.5, -3.], Plate(Rectangle(1., 1.), 0.1))]
    for pos, shape in extra[:max(0, n_obstacles - 2)]:
        environment.add_obstacle(Obstacle({'position': pos}, shape=shape))
    opts = {'horizon_time': 5.}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def config_quadrotor2d(options=None, build_solver=True):
    """examples/p2p_quadrotor.py: planar Quadrotor, one tall Rectangle wall,
    safety distance 0.1, horizon 5 s; rows of degree 3 (n=154, m=615)."""
    from . import Quadrotor
    vehicle = Quadrotor()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-4., -4., 0., 0., 0.])
    vehicle.set_terminal_conditions([4., 4.])
    environment = Environment(room={'shape': Square(10.)})
    environment.add_obstacle(Obstacle({'position': [-0.6, -5.4]},
                                      shape=Rectangle(width=0.2, height=12.)))
    opts = {'horizon_time': 5}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def config_dubins(options=None, build_solver=True, substitution=True, exact=False,
                  shape=None, knot_intervals=None):
    """examples/p2p_dubins.py with a fixed end time: Dubins(vmax 0.7, |w| <= pi/3,
    substitution as in the example; substitution=False is the vehicle's default
    formulation, dubins.py:63), Square(5) room centred at (1.5, 1.5), one Circle(0.5)
    obstacle drifting in x; horizon 10 s."""
    from . import Dubins
    vehicle = Dubins(shapes=shape,
                     bounds={'vmax': 0.7, 'wmax': np.pi / 3., 'wmin': -np.pi / 3.},
                     options={'substitution': substitution, 'exact_substitution': exact})
    if knot_intervals is not None:
        vehicle.define_knots(knot_intervals=knot_intervals)
    vehicle.set_initial_conditions([0., 0., 0.])
    vehicle.set_terminal_conditions([3., 3., 0.])
    environment = Environment(room={'shape': Square(5.), 'position': [1.5, 1.5]})
    trajectories = {'velocity': {'time': [0.5], 'values': [[0.25, 0.0]]}}
    environment.add_obstacle(Obstacle({'position': [1., 1.]}, shape=Circle(0.5),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver)


def config_dubins_plain(options=None, build_solver=True):
    """The Dubins vehicle's default formulation (substitution=False, dubins.py:63): the
    integrated position enters the terminal and collision rows directly."""
    return config_dubins(options, build_solver, substitution=False)


def config_dubins_rect(options=None, build_solver=True):
    """Dubins with a rectangular shape, default formulation: the heading tan(theta/2)
    enters the collision rows (vehicle.py:122-177 with tg_ha), degree-4 rows with an
    intermediate factor."""
    from . import Rectangle
    return config_dubins(options, build_solver, substitution=False,
                         shape=Rectangle(width=0.4, height=0.2), knot_intervals=5)


def config_dubins_exact(options=None, build_solver=True):
    """Dubins with exact_substitution: dx, dy on the product basis, equality rows."""
    return config_dubins(options, build_solver, substitution=True, exact=True,
                         knot_intervals=5)


def config_bicycle(options=None, build_solver=True):
    """examples/p2p_bicycle.py with a fixed end time: Bicycle(length 0.4, no substitution,
    5 knot intervals) from (0, 0, 0, delta 0) to (3, 3, 0), Square(5) room centred at
    (1.5, 1.5), one Circle(0.5) obstacle drifting in x."""
    from . import Bicycle
    vehicle = Bicycle(length=0.4, options={'plot_type': 'car', 'substitution': False})
    vehicle.define_knots(knot_intervals=5)
    vehicle.set_initial_conditions([0., 0., 0., 0.])
    vehicle.set_terminal_conditions([3., 3., 0.])
    environment = Environment(room={'shape': Square(5.), 'position': [1.5, 1.5]})
    trajectories = {'velocity': {'time': [0.5], 'values': [[0.3, 0.0]]}}
    environment.add_obstacle(Obstacle({'position': [1., 1.]}, shape=Circle(0.5),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver)


def config_agv(options=None, build_solver=True):
    """examples/p2p_agv.py with a fixed end time: AGV(length 0.8, Rectangle(0.8, 0.2), 5 knot
    intervals) parking between two rectangles in a Rectangle(4, 1) corridor."""
    from . import AGV, Rectangle
    vehicle = AGV(length=0.8, options={'plot_type': 'agv'})
    vehicle.define_knots(knot_intervals=5)
    vehicle.set_initial_conditions([0.8, -0.05, 0., 0.])
    vehicle.set_terminal_conditions([2.45, -0.35, 0.])
    environment = Environment(room={'shape': Rectangle(width=4, height=1), 'position': [2, 0.]})
    rectangle = Rectangle(width=0.8, height=0.2)
    environment.add_obstacle(Obstacle({'position': [1., -0.35]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [3.4, -0.35]}, shape=rectangle))
    return _p2p(vehicle, environment, options, build_solver)


def config_quadrotor3d_simple(options=None, build_solver=True):
    """SimpleQuadrotor3D (position splines of degree 4, quadratic thrust / rate / tilt rows)
    in the scene of examples/p2p_3dquadrotor.py: Cuboid(8, 6, 8) room, two plates, the second
    one moving down; horizon 10 s.  (No reference example uses this model.)"""
    from . import SimpleQuadrotor3D, Cuboid, Plate, Rectangle
    vehicle = SimpleQuadrotor3D(0.5)
    vehicle.set_initial_conditions([-3, -2, -0.5, 0, 0, 0, 0, 0])
    vehicle.set_terminal_conditions([3, 2, 0.5])
    vehicle.set_options({'safety_distance': 0.1, 'safety_weight': 10})
    environment = Environment(room={'shape': Cuboid(8, 6, 8)})
    plate = lambda: Plate(Rectangle(5., 8.), 0.1, orientation=[0., np.pi / 2, 0.])
    trajectory = {'velocity': {'time': [1.5], 'values': [[0, 0, -0.6]]}}
    environment.add_obstacle(Obstacle({'position': [-2, 0, -2]}, shape=plate()))
    environment.add_obstacle(Obstacle({'position': [2, 0, 3.5]}, shape=plate(),
                                      simulation={'trajectories': trajectory}))
    return _p2p(vehicle, environment, options, build_solver)


def config_holonomic_orient(options=None, build_solver=True):
    """examples/p2p_holonomic_orient.py with a fixed end time: HolonomicOrient
    (Rectangle(0.2, 0.4), heading free, norm-1 regularisation of the heading rate),
    Square(5) room, two Rectangle(3, 0.2) walls and a moving Circle(0.4)."""
    from . import HolonomicOrient, Rectangle
    vehicle = HolonomicOrient()
    vehicle.set_options({'reg_type': 'norm_1', 'reg_weight': 10})
    vehicle.set_initial_conditions([-1.5, -1.5, np.pi / 4.])
    vehicle.set_terminal_conditions([2., 2., np.pi / 2.])
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-1.8, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    trajectories = {'velocity': {'time': [3., 4.], 'values': [[-0.15, 0.0], [0., 0.15]]}}
    environment.add_obstacle(Obstacle({'position': [1.5, 0.5]}, shape=Circle(0.4),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver)


def config_disturbances(options=None, build_solver=True):
    """examples/p2p_holonomic_disturbances.py: Holonomic with a first-order actuator lag
    (time_constant 0.1) and a filtered input disturbance (fc 0.01, stdev 0.05), stop_tol 1e-2,
    Square(5) room, two Rectangle(3, 0.2) walls and a Circle(0.4) that starts moving at t = 3 s.
    The example keeps the reference's non-ideal vehicle defaults, so they are set here: the
    closed loop runs in execution/batch_mpc.py (the host Vehicle.predict is ideal only)."""
    vehicle = Holonomic()
    vehicle.set_options({'safety_distance': 0.1, '1storder_delay': True, 'time_constant': 0.1,
                         'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)},
                         'stop_tol': 1.e-2, 'ideal_prediction': False, 'ideal_update': False})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2.1, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    trajectories = {'velocity': {'time': [3., 4.], 'values': [[-0.15, 0.0], [0., 0.15]]}}
    environment.add_obstacle(Obstacle({'position': [1.5, 0.5]}, shape=Circle(0.4),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver)


def config_freeT(options=None, build_solver=True, moving=False):
    """Minimum-time variant of examples/p2p_holonomic.py (freeT=True, the
    example's commented alternative): two rectangular walls and a circle
    (moving as in the example if ``moving``), T is a decision variable
    (n=126, m=622, rows of degree 3)."""
    vehicle = Holonomic()
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2.1, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    trajectories = {'velocity': {'time': [3., 4.],
                                 'values': [[-0.15, 0.0], [0., 0.15]]}}
    environment.add_obstacle(Obstacle(
        {'position': [1.5, 0.5]}, shape=Circle(0.4),
        simulation={'trajectories': trajectories} if moving else None))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_freeT_moving(options=None, build_solver=True):
    return config_freeT(options, build_solver, moving=True)


def config_freeT_safety(options=None, build_solver=True):
    """Minimum-time problem with a safety-distance slack (examples/p2p_holonomic.py with
    freeT=True): the relative start t/T of the slack objective is 0 for a free end time."""
    vehicle = Holonomic()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    environment.add_obstacle(Obstacle({'position': [0.3, 0.2]}, shape=Circle(0.5)))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_dubins_freeT(options=None, build_solver=True, init_v_til=0.):
    """examples/p2p_dubins.py as written: substitution, 5 knot intervals, free end time (the
    motion time multiplies the integrated velocity: T x intermediate cross terms).
    ``init_v_til`` > 0 replaces the reference's zero-speed initial guess (vehicle option)."""
    from . import Dubins
    vehicle = Dubins(bounds={'vmax': 0.7, 'wmax': np.pi / 3., 'wmin': -np.pi / 3.},
                     options={'substitution': True, 'init_v_til': init_v_til})
    vehicle.define_knots(knot_intervals=5)
    vehicle.set_initial_conditions([0., 0., 0.])
    vehicle.set_terminal_conditions([3., 3., 0.])
    environment = Environment(room={'shape': Square(5.), 'position': [1.5, 1.5]})
    trajectories = {'velocity': {'time': [0.5], 'values': [[0.25, 0.0]]}}
    environment.add_obstacle(Obstacle({'position': [1., 1.]}, shape=Circle(0.5),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_holonomic_orient_freeT(options=None, build_solver=True):
    """examples/p2p_holonomic_orient.py as written: the scene of config_holonomic_orient with a free
    end time (n=151, m=2961, n_par=55)."""
    from . import HolonomicOrient, Rectangle
    vehicle = HolonomicOrient()
    vehicle.set_options({'reg_type': 'norm_1', 'reg_weight': 10})
    vehicle.set_initial_conditions([-1.5, -1.5, np.pi / 4.])
    vehicle.set_terminal_conditions([2., 2., np.pi / 2.])
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-1.8, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    trajectories = {'velocity': {'time': [3., 4.], 'values': [[-0.15, 0.0], [0., 0.15]]}}
    environment.add_obstacle(Obstacle({'position': [1.5, 0.5]}, shape=Circle(0.4),
                                      simulation={'trajectories': trajectories}))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_quadrotor2d_freeT(options=None, build_solver=True):
    """The scene of config_quadrotor2d (examples/p2p_quadrotor.py) with a free end time
    (n=76, m=443, n_par=27)."""
    from . import Quadrotor
    vehicle = Quadrotor()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-4., -4., 0., 0., 0.])
    vehicle.set_terminal_conditions([4., 4.])
    environment = Environment(room={'shape': Square(10.)})
    environment.add_obstacle(Obstacle({'position': [-0.6, -5.4]},
                                      shape=Rectangle(width=0.2, height=12.)))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_quadrotor3d_simple_freeT(options=None, build_solver=True):
    """The scene of config_quadrotor3d_simple with a free end time (n=159, m=833, n_par=63)."""
    from . import SimpleQuadrotor3D, Cuboid, Plate, Rectangle
    vehicle = SimpleQuadrotor3D(0.5)
    vehicle.set_initial_conditions([-3, -2, -0.5, 0, 0, 0, 0, 0])
    vehicle.set_terminal_conditions([3, 2, 0.5])
    vehicle.set_options({'safety_distance': 0.1, 'safety_weight': 10})
    environment = Environment(room={'shape': Cuboid(8, 6, 8)})
    plate = lambda: Plate(Rectangle(5., 8.), 0.1, orientation=[0., np.pi / 2, 0.])
    trajectory = {'velocity': {'time': [1.5], 'values': [[0, 0, -0.6]]}}
    environment.add_obstacle(Obstacle({'position': [-2, 0, -2]}, shape=plate()))
    environment.add_obstacle(Obstacle({'position': [2, 0, 3.5]}, shape=plate(),
                                      simulation={'trajectories': trajectory}))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_trailer(options=None, build_solver=True, init_v_til=0.):
    """examples/p2p_trailer.py: a Dubins vehicle (Circle(0.2), 9 knot intervals) pulling a
    Rectangle(0.2, 0.2) trailer on a 0.6 m hitch from (0, 0, 0) to (3.4, 3, 0), trailer heading
    0 -> 0, empty Square(5) room, free end time; as in the example the lead vehicle is added
    to the problem as a child and as a vehicle of its own."""
    from . import Dubins, Trailer, Rectangle
    vehicle = Dubins(shapes=Circle(0.2), bounds={'vmax': 0.8, 'wmax': np.pi / 3., 'wmin': -np.pi / 3.},
                     options={'init_v_til': init_v_til})
    vehicle.define_knots(knot_intervals=9)
    vehicle.set_initial_conditions([0., 0., 0.])
    vehicle.set_terminal_conditions([3.4, 3., 0.])
    trailer = Trailer(lead_veh=vehicle, shapes=Rectangle(0.2, 0.2), l_hitch=0.6,
                      bounds={'tmax': np.pi / 4., 'tmin': -np.pi / 4.})
    trailer.define_knots(knot_intervals=9)
    trailer.set_initial_conditions(0.)
    trailer.set_terminal_conditions(0.)
    environment = Environment(room={'shape': Square(5.), 'position': [1.5, 1.5]})
    opts = {'verbose': 0}
    opts.update(options or {})
    problem = Point2point(trailer, environment, options=opts, freeT=True)
    problem.father.add(vehicle)
    problem.vehicles.append(vehicle)
    vehicle.to_simulate = False
    if build_solver:
        problem.init()
    else:
        f = problem.father
        f.reset()
        problem.construct()
        f.translate_symbols()
        f.construct_variables()
        f.construct_parameters()
        rows, lb, ub = f.construct_constraints()
        from .basics.lowering import lower
        f.tables = lower(f._var_ids, f._par_ids, rows, f.construct_objective(), lb, ub, f.order_hint())
        f.init_variables()
        f.init_parameters()
        f.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
    problem.reinitialize()
    return problem


def config_warehouse(options=None, build_solver=True):
    """examples/p2p_holonomic_warehouse.py: Holonomic with Euclidean speed / acceleration limits
    and a safety distance, six square racks and two moving circles in a 7 x 4.5 room, free
    end time (n = 395, m = 1628).  The cold start from the straight line through the racks is
    hard: the oracle ends in Restoration_Failed after ~700 iterations (feasibility phase
    included) and converges with the solver option retry_mu = 1e-3 (T = 23.5 s)."""
    vehicle = Holonomic(options={'syslimit': 'norm_2', 'safety_distance': 0.1})
    vehicle.define_knots(knot_intervals=10)
    vehicle.set_initial_conditions([0., 0.])
    vehicle.set_terminal_conditions([6., 3.5])
    environment = Environment(room={'shape': Rectangle(width=7., height=4.5), 'position': [3., 1.75]})
    rectangle = Rectangle(width=1., height=1.)
    for pos in ([1., 1.], [3., 1.], [5., 1.], [1., 2.5], [3., 2.5], [5., 2.5]):
        environment.add_obstacle(Obstacle({'position': pos}, shape=rectangle))
    trajectories1 = {'velocity': {'time': [0, 2], 'values': [[0., 0.0], [0., 0.15]]}}
    trajectories2 = {'velocity': {'time': [0, 2], 'values': [[0., 0.0], [0., -0.1]]}}
    environment.add_obstacle(Obstacle({'position': [4., 2.5]}, shape=Circle(0.5),
                                      simulation={'trajectories': trajectories2}))
    environment.add_obstacle(Obstacle({'position': [2., 1.]}, shape=Circle(0.5),
                                      simulation={'trajectories': trajectories1}))
    return _p2p(vehicle, environment, options, build_solver, freeT=True)


def config_revolving_door_diffdrive(options=None, build_solver=True, init_v_til=0.):
    """examples/revolving_door_diffdrive.py: a Dubins vehicle (default formulation, 6 knot
    intervals) through the slowly revolving door: two static and two rotating beams,
    horizon 15 s, hard terminal constraints."""
    from . import Dubins, Beam
    vehicle = Dubins(bounds={'vmax': 0.7, 'wmin': -30., 'wmax': 30.}, options={'init_v_til': init_v_til})
    vehicle.define_knots(knot_intervals=6)
    vehicle.set_initial_conditions([0., -2.0, np.pi / 2])
    vehicle.set_terminal_conditions([-1.5, 2.0, np.pi / 2])
    environment = Environment(room={'shape': Square(5.)})
    beam1 = Beam(width=2.2, height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2., 0.]}, shape=beam1))
    environment.add_obstacle(Obstacle({'position': [2., 0.]}, shape=beam1))
    beam2 = Beam(width=1.4, height=0.2)
    horizon_time = 15.
    omega = 0.1 * 1. * (2 * np.pi / horizon_time)
    for orient in (0. + np.pi / 4., 0.5 * np.pi + np.pi / 4.):
        environment.add_obstacle(Obstacle(
            {'position': [0., 0.], 'velocity': [0., 0.], 'orientation': orient,
             'angular_velocity': omega}, shape=beam2, simulation={},
            options={'horizon_time': horizon_time}))
    opts = {'horizon_time': horizon_time, 'hard_term_con': True}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def config_revolving_door_quadrotor(options=None, build_solver=True):
    """examples/revolving_door_quadrotor.py: the planar Quadrotor (radius 0.1, u1max 10) through
    the revolving door -- two static and two rotating beams (omega = 0.45 rev / horizon),
    horizon 10 s."""
    from . import Quadrotor, Beam
    vehicle = Quadrotor(radius=0.1, bounds={'u1max': 10, 'u2max': 8})
    vehicle.define_knots(knot_intervals=10)
    vehicle.set_initial_conditions([0., -2.0])
    vehicle.set_terminal_conditions([-0.5, 2.0])
    environment = Environment(room={'shape': Square(5.)})
    beam1 = Beam(width=2.2, height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2., 0.]}, shape=beam1))
    environment.add_obstacle(Obstacle({'position': [2., 0.]}, shape=beam1))
    beam2 = Beam(width=1.4, height=0.2)
    horizon_time = 10.
    omega = 0.45 * 1. * (2 * np.pi / horizon_time)
    for orient in (0. + np.pi / 4, 0.5 * np.pi + np.pi / 4):
        environment.add_obstacle(Obstacle(
            {'position': [0., 0.], 'velocity': [0., 0.], 'orientation': orient,
             'angular_velocity': omega}, shape=beam2, simulation={},
            options={'horizon_time': horizon_time}))
    opts = {'horizon_time': horizon_time}
    opts.update(options or {})
    return _p2p(vehicle, environment, opts, build_solver)


def instance_data(problem, batch, jitter=0.0, seed=0, current_time=0.):
    """(X0[B,n], P[B,n_par]) for a cold solve: linear initial guess
    (holonomic.py:118-127) and parameters at current_time.  jitter>0 perturbs
    state0/poseT by U(-jitter,jitter) and obstacle positions by U(-j/2, j/2)
    (SURVEY.md section 8d)."""
    f = problem.father
    rng = np.random.default_rng(seed)
    vehicle = problem.vehicles[0]
    state0 = np.array(vehicle.prediction['state'], dtype=float)
    goal = 'poseT' if hasattr(vehicle, 'poseT') else 'positionT'   # SimpleQuadrotor3D
    poseT = np.array(getattr(vehicle, goal), dtype=float)
    obst0 = [o.signals['position'][:, -1].copy()
             for o in problem.environment.obstacles]
    X0 = np.zeros((batch, f.tables.n))
    P = np.zeros((batch, f.tables.n_par))
    for b in range(batch):
        if jitter > 0. and b > 0:
            vehicle.prediction['state'] = state0 + rng.uniform(-jitter, jitter, len(state0))
            setattr(vehicle, goal, poseT + rng.uniform(-jitter, jitter, len(poseT)))
            for o, p0 in zip(problem.environment.obstacles, obst0):
                o.signals['position'][:, -1] = p0 + rng.uniform(
                    -0.5 * jitter, 0.5 * jitter, len(p0))
        problem.reinitialize()
        X0[b] = f.get_variables().cat
        P[b] = f.set_parameters(current_time).cat
    vehicle.prediction['state'] = state0
    setattr(vehicle, goal, poseT)
    for o, p0 in zip(problem.environment.obstacles, obst0):
        o.signals['position'][:, -1] = p0
    problem.reinitialize()
    return X0, P


def config_free_end(options=None, build_solver=True):
    """FreeEndPoint2point (the agent problem of a RendezVous): config 1's scene with the
    terminal position as decision variables conT0."""
    from .problems.point2point import FreeEndPoint2point
    vehicle = Holonomic()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = Environment(room={'shape': Square(5.)})
    environment.add_obstacle(Obstacle({'position': [1.5, -1]}, shape=Circle(0.5)))
    opts = {'verbose': 0}
    opts.update(options or {})
    problem = FreeEndPoint2point(vehicle, environment, opts, {vehicle: [0, 1]})
    if build_solver:
        problem.init()
    else:
        f = problem.father
        f.reset()
        problem.construct()
        f.translate_symbols()
        f.construct_variables()
        f.construct_parameters()
        rows, lb, ub = f.construct_constraints()
        from .basics.lowering import lower
        f.tables = lower(f._var_ids, f._par_ids, rows, f.construct_objective(), lb, ub, f.order_hint())
        f.init_variables()
        f.init_parameters()
        f.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
    problem.reinitialize()
    return problem


def config_interveh(options=None, build_solver=True, start_offset=0.):
    """examples/p2p_holonomic_interveh_avoidance.py: two Holonomic vehicles swapping places
    across an empty Square(5) room, one NLP, separating hyperplanes between the vehicles
    (Environment.define_intervehicle_collision_constraints).  start_offset moves vehicle 0's
    start off the head-on line (config_interveh_offset)."""
    N = 2
    vehicles = [Holonomic() for _ in range(N)]
    for k, vehicle in enumerate(vehicles):
        vehicle.set_initial_conditions([1.5 * np.cos((k * 2. * np.pi) / N),
                                        1.5 * np.sin((k * 2. * np.pi) / N) + (start_offset if k == 0 else 0.)])
        vehicle.set_terminal_conditions([-1.5 * np.cos((k * 2. * np.pi) / N),
                                         -1.5 * np.sin((k * 2. * np.pi) / N)])
    environment = Environment(room={'shape': Square(5.)})
    opts = {'inter_vehicle_avoidance': True}
    opts.update(options or {})
    return _p2p(vehicles, environment, opts, build_solver)


def config_interveh_offset(options=None, build_solver=True):
    """config_interveh with vehicle 0 starting 0.1 m off the head-on line: with the symmetric
    start, rounding decides on which side the vehicles pass each other."""
    return config_interveh(options, build_solver, start_offset=0.1)


def config_formation_central_example(options=None, build_solver=True):
    """examples/formation_holonomic_central.py exactly: soft formation AND inter-vehicle
    avoidance (six vehicle pairs, each with a separating hyperplane spline)."""
    opts = {'inter_vehicle_avoidance': True}
    opts.update(options or {})
    return config_formation_central(opts, build_solver)


def config_formation_central(options=None, build_solver=True, soft=True):
    """examples/formation_holonomic_central.py: four Holonomic vehicles starting in a row,
    formation RegularPolyhedron(0.2, 4) to (2, 2), two Rectangle(3, 0.2) walls, horizon 15 s,
    soft formation constraints with weight 100 (option inter_vehicle_avoidance as in the
    example: config_formation_central_example)."""
    from .vehicles.fleet import Fleet
    from .basics.shape import RegularPolyhedron
    from .problems.formation_central import FormationPoint2pointCentral
    N = 4
    vehicles = [Holonomic() for _ in range(N)]
    for k, vehicle in enumerate(vehicles):
        vehicle.set_initial_conditions([-1. - 0.5 * N * 0.5 + 0.5 * k, -1.5])
    fleet = Fleet(vehicles)
    configuration = RegularPolyhedron(0.2, N, np.pi / 4.).vertices.T
    fleet.set_configuration(configuration.tolist())
    fleet.set_terminal_conditions((np.array([2., 2.]) + configuration).tolist())
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-1.8, 0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, 0.5]}, shape=rectangle))
    opts = {'verbose': 0, 'horizon_time': 15, 'soft_formation': soft,
            'soft_formation_weight': 100}
    opts.update(options or {})
    problem = FormationPoint2pointCentral(fleet, environment, options=opts)
    if build_solver:
        problem.init()
    else:
        problem.father.reset()
        problem.construct()
        f = problem.father
        f.translate_symbols()
        f.construct_variables()
        f.construct_parameters()
        rows, lb, ub = f.construct_constraints()
        from .basics.lowering import lower
        f.tables = lower(f._var_ids, f._par_ids, rows, f.construct_objective(), lb, ub,
                         f.order_hint())
        f.init_variables()
        f.init_parameters()
        f.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
    problem.reinitialize()
    return problem


def config3(n_agents=4, options=None, build_solver=True, rank=0, world=1, group=None,
            interconnection='circular'):
    """FormationPoint2point ADMM (examples/formation_holonomic.py scaled to
    n_agents, 2 rectangular obstacles as in the C++ formation test): agents on
    a circle of radius 0.2, circular interconnection, rho = 1."""
    from .vehicles.fleet import Fleet
    from .basics.shape import RegularPolyhedron
    from .problems.admm import FormationPoint2point
    vehicles = [Holonomic() for _ in range(n_agents)]
    fleet = Fleet(vehicles, interconnection=interconnection)
    if n_agents == 4:
        configuration = RegularPolyhedron(0.2, n_agents, np.pi / 4.).vertices.T
    else:
        ang = 2 * np.pi * np.arange(n_agents) / n_agents
        configuration = 0.2 * np.c_[np.cos(ang), np.sin(ang)]
    init_positions = np.array([-1.5, -1.5]) + configuration
    terminal_positions = np.array([2., 2.]) + configuration
    fleet.set_configuration(configuration.tolist())
    fleet.set_initial_conditions(init_positions.tolist())
    fleet.set_terminal_conditions(terminal_positions.tolist())
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2.1, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    opts = {'rho': 1., 'horizon_time': 10, 'verbose': 0}
    opts.update(options or {})
    problem = FormationPoint2point(fleet, environment, options=opts, rank=rank,
                                   world=world, group=group)
    problem.init(build_solver=build_solver)
    return problem


def config_rendezvous(n_agents=4, options=None, build_solver=True, rank=0, world=1, group=None):
    """RendezVous (problems/admm.py; reference rendezvous.py, examples/
    rendezvous_holonomic_export.py scaled to n_agents): Holonomic vehicles starting in the
    corners of the room agree by ADMM on where to meet -- in a RegularPolyhedron(0.2)
    configuration around a common centre; each agent only proposes its own terminal
    position."""
    from .vehicles.fleet import Fleet
    from .basics.shape import RegularPolyhedron
    from .problems.admm import RendezVous
    vehicles = [Holonomic() for _ in range(n_agents)]
    fleet = Fleet(vehicles)
    ang = 2 * np.pi * np.arange(n_agents) / n_agents + np.pi / 4.
    configuration = 0.2 * np.c_[np.cos(ang), np.sin(ang)]
    init_positions = 1.8 * np.c_[np.cos(ang), np.sin(ang)] * np.array([1., 0.8])
    terminal_positions = 0.5 * init_positions          # first proposals: half way to the middle
    fleet.set_configuration(configuration.tolist())
    fleet.set_initial_conditions(init_positions.tolist())
    fleet.set_terminal_conditions(terminal_positions.tolist())
    environment = Environment(room={'shape': Square(5.)})
    environment.add_obstacle(Obstacle({'position': [0.9, 0.1]}, shape=Circle(0.3)))
    opts = {'rho': 3., 'horizon_time': 10, 'verbose': 0}
    opts.update(options or {})
    problem = RendezVous(fleet, environment, options=opts, rank=rank, world=world, group=group)
    problem.init(build_solver=build_solver)
    return problem


def config_formation_dd(n_agents=4, options=None, build_solver=True, rank=0, world=1, group=None):
    """The formation of config 3 solved by dual decomposition (reference formation_dualdec.py;
    the method the reference compares with ADMM in examples/compare_distributed_optimization_
    quadrotors.py): every agent's NLP holds its own trajectory and copies of its two
    neighbours', coupled by hard formation rows; dual ascent with step rho."""
    from .vehicles.fleet import Fleet
    from .basics.shape import RegularPolyhedron
    from .problems.dualdecomposition import FormationPoint2pointDualDecomposition
    vehicles = [Holonomic() for _ in range(n_agents)]
    fleet = Fleet(vehicles, interconnection='circular')
    if n_agents == 4:
        configuration = RegularPolyhedron(0.2, n_agents, np.pi / 4.).vertices.T
    else:
        ang = 2 * np.pi * np.arange(n_agents) / n_agents
        configuration = 0.2 * np.c_[np.cos(ang), np.sin(ang)]
    fleet.set_configuration(configuration.tolist())
    fleet.set_initial_conditions((np.array([-1.5, -1.5]) + configuration).tolist())
    fleet.set_terminal_conditions((np.array([2., 2.]) + configuration).tolist())
    environment = Environment(room={'shape': Square(5.)})
    rectangle = Rectangle(width=3., height=0.2)
    environment.add_obstacle(Obstacle({'position': [-2.1, -0.5]}, shape=rectangle))
    environment.add_obstacle(Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    opts = {'rho': 0.5, 'horizon_time': 10, 'verbose': 0}
    opts.update(options or {})
    problem = FormationPoint2pointDualDecomposition(fleet, environment, options=opts, rank=rank,
                                                    world=world, group=group)
    problem.init(build_solver=build_solver)
    return problem
