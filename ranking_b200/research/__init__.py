"""Research models of the reference (tensorflow_ranking/research), on the sm_90a kernels."""
from ranking_b200.research import dasalc  # noqa: F401
