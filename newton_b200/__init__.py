"""newton_b200 - H100-native batched rigid-body stepper behind Newton's solver API."""
from .sim import (  # noqa: F401
    MAXVAL, BodyFlags, Contacts, Control, GeoType, JointDofConfig, JointType, Model, ModelBuilder,
    ModelFlags, ShapeConfig, ShapeFlags, State, StateFlags, eval_fk, eval_ik, eval_inverse_dynamics_force,
    eval_inverse_dynamics_passive, eval_jacobian, eval_mass_matrix,
)
from .sim.collide import CollisionPipeline, SpeculativeContactConfig  # noqa: F401,E402
from . import solvers  # noqa: F401,E402
from . import selection  # noqa: F401,E402
from . import sensors  # noqa: F401,E402
