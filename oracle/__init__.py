"""oracle/ -- CPU restatement (NumPy/SciPy fp64) of akopich/spark-gp's algorithm.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` leg may import anything under `oracle/`.  The product
package (`spark_gp_b200/`) never imports it and fails loudly when its CUDA
extension is missing.

Every function cites the reference file:line (relative to the reference's
`src/main/scala/org/apache/spark/ml/`) it follows.  The reference is Scala on
Breeze + netlib LAPACK; there is no JVM in this image (nor on the GPU box), so
the reference itself cannot be executed.  The restatement is pinned on the
only known-answer vectors the reference's own tests hold for this path
(`src/test/.../RBFKernelTest.scala:31-38,62-76`: RBF 3x3 matrix and crossKernel
rows) and on its analytic-vs-numeric derivative tests
(`RBFKernelTest.scala:51-60`, `ARDRBFKernelTest.scala:21-31`).  Nothing in the
reference pins G, b, magicVector, magicMatrix, mean or variance: for those the
restatement *is* the parity definition (DESIGN.md says so).

Third-party arithmetic the reference delegates to and how it is restated:
  * Breeze `DenseMatrix * DenseMatrix` / `* DenseVector`  -> BLAS dgemm/dgemv (numpy @).
  * Breeze `A \\ b` (square)                               -> LAPACK dgesv  (scipy lu_factor/lu_solve).
  * Breeze `inv(A)`                                        -> dgetrf+dgetri (scipy.linalg.inv).
  * Breeze `eigSym(A).eigenvalues`                         -> dsyevd        (scipy eigvalsh, driver='evd').
  * Breeze `cholesky(B)`                                   -> dpotrf (lower).
  * `logDetAndInv` (commons/util/logDetAndInv.scala:58-63) -> dgetrf + dgetri.
Versions are unpinned in the reference (transitive deps of spark-mllib 3.1.1,
`build.sbt:5-13`); the algorithms are the standard LAPACK ones.
"""
from .kernels import (Kernel, ARDRBFKernel, RBFKernel, EyeKernel, ConstantTimesKernel,
                      TrainableScalarTimesKernel, SumOfKernels, Scalar, WhiteNoiseKernel,
                      TrainingVectorsNotInitializedException, const)
from .ppa import (get_matrix_kmn_knm_and_vector_kmny, get_magic_vector, tail_errors,
                  NotPositiveDefiniteException, GaussianProjectedProcessRawPredictor,
                  get_kernel, group_for_experts, get_expert_labels_and_kernels,
                  projected_process)
from .regression import regression_likelihood_and_gradient, log_det_and_inv
from .scaling import scale
