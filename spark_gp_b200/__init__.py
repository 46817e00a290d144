"""spark_gp_b200 -- H100-native projected-process (sparse GP) hot path behind the reference's API.

Only what the path needs: `csrc/` (CUDA kernels + the C-ABI of include/sgp.h), the ctypes binding, and a
host-side mirror of the reference's kernel DSL / Estimator surface.  No CPU fallback."""
from .kernels import (Kernel, ARDRBFKernel, RBFKernel, EyeKernel, ConstantTimesKernel, TrainableScalarTimesKernel,
                      SumOfKernels, Scalar, WhiteNoiseKernel, const)
from .engine import (ProjectedProcessEngine, NotPositiveDefiniteException, TrainingVectorsNotInitializedException,
                     MatrixSingularException, SgpError, OperandRangeError)
from .regression import (GaussianProcessRegression, GaussianProcessRegressionModel, RandomActiveSetProvider,
                         GreedilyOptimizingActiveSetProvider, KMeansActiveSetProvider)
from .classification import GaussianProcessClassifier, GaussianProcessClassificationModel, OneVsRest, OneVsRestModel
from .utils import scale
from .tuning import (BinaryClassificationEvaluator, CrossValidator, CrossValidatorModel, ParamGridBuilder,
                     RegressionEvaluator, MulticlassClassificationEvaluator, TrainValidationSplit,
                     TrainValidationSplitModel)
