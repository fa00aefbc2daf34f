from .function import (  # noqa: F401
    AugmentedExpectedImprovement,
    augmented_expected_improvement,
    BatchMonteCarloExpectedImprovement,
    ExpectedImprovement,
    LogExpectedImprovement,
    MinValueEntropySearch,
    MonteCarloExpectedImprovement,
    MultipleOptimismNegativeLowerConfidenceBound,
    multiple_optimism_lower_confidence_bound,
    monte_carlo_expected_improvement,
    min_value_entropy_search,
    NegativeLowerConfidenceBound,
    ProbabilityOfFeasibility,
    ProbabilityOfImprovement,
    batch_monte_carlo_expected_improvement,
    expected_improvement,
    log_expected_improvement,
    lower_confidence_bound,
    probability_below_threshold,
)
from .greedy_batch import (  # noqa: F401
    Fantasizer,
    LocalPenalization,
    PenalizedAcquisition,
    hard_local_penalizer,
    local_penalizer,
    soft_local_penalizer,
)
from .interface import (  # noqa: F401
    AcquisitionFunctionBuilder,
    GreedyAcquisitionFunctionBuilder,
    SingleModelAcquisitionBuilder,
    SingleModelGreedyAcquisitionBuilder,
    SingleModelVectorizedAcquisitionBuilder,
    VectorizedAcquisitionFunctionBuilder,
)
from .utils import split_acquisition_function, split_acquisition_function_calls  # noqa: F401
