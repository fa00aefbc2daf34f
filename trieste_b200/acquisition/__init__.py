from .active_learning import (  # noqa: F401
    BayesianActiveLearningByDisagreement,
    ExpectedFeasibility,
    PredictiveVariance,
    bayesian_active_learning_by_disagreement,
    bichon_ranjan_criterion,
    predictive_variance,
)
from .combination import Product, Reducer, Sum  # noqa: F401
from .continuous_thompson_sampling import (  # noqa: F401
    GreedyContinuousThompsonSampling,
    ParallelContinuousThompsonSampling,
    negate_trajectory_function,
)
from .function import (  # noqa: F401
    AugmentedExpectedImprovement,
    augmented_expected_improvement,
    BatchExpectedImprovement,
    BatchMonteCarloExpectedImprovement,
    ExpectedImprovement,
    GIBBON,
    GibbonAcquisition,
    LogExpectedImprovement,
    MakePositive,
    MinValueEntropySearch,
    MonteCarloExpectedImprovement,
    MultipleOptimismNegativeLowerConfidenceBound,
    multiple_optimism_lower_confidence_bound,
    monte_carlo_expected_improvement,
    min_value_entropy_search,
    NegativeLowerConfidenceBound,
    ProbabilityOfFeasibility,
    ProbabilityOfImprovement,
    batch_expected_improvement,
    batch_monte_carlo_expected_improvement,
    expected_improvement,
    gibbon_quality_term,
    gibbon_repulsion_term,
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
from .multi_objective import (  # noqa: F401
    HIPPO,
    ExpectedHypervolumeImprovement,
    expected_hv_improvement,
    hippo_penalized_ehvi,
    hippo_penalizer,
)
from .interface import (  # noqa: F401
    AcquisitionFunctionBuilder,
    GreedyAcquisitionFunctionBuilder,
    SingleModelAcquisitionBuilder,
    SingleModelGreedyAcquisitionBuilder,
    SingleModelVectorizedAcquisitionBuilder,
    VectorizedAcquisitionFunctionBuilder,
)
from .utils import (  # noqa: F401
    MultivariateNormalCDF,
    select_nth_output,
    split_acquisition_function,
    split_acquisition_function_calls,
)
