"""Multi-objective geometry on the host (Pareto dominance, fronts, hypervolume, non-dominated partitions), the expected
hypervolume improvement and HIPPO's greedy batches over it, whose per-candidate work runs on the device."""
from .dominance import non_dominated  # noqa: F401
from .function import (  # noqa: F401
    HIPPO,
    ExpectedHypervolumeImprovement,
    expected_hv_improvement,
    hippo_penalized_ehvi,
    hippo_penalizer,
)
from .pareto import Pareto, get_reference_point  # noqa: F401
from .partition import (  # noqa: F401
    DividedAndConquerNonDominated,
    ExactPartition2dNonDominated,
    prepare_default_non_dominated_partition_bounds,
)
