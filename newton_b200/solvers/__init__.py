from .featherstone import SolverFeatherstone
from .semi_implicit import SolverSemiImplicit
from .solver import SolverBase
from .xpbd import SolverXPBD

__all__ = ["SolverBase", "SolverFeatherstone", "SolverSemiImplicit", "SolverXPBD"]
