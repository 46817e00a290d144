package org.apache.spark.ml.commons

import breeze.linalg.{DenseMatrix => BDM, DenseVector => BDV}
import org.apache.spark.ml.commons.kernel._
import org.apache.spark.ml.linalg.Vector
import org.apache.spark.rdd.RDD

/** JNI binding of libsgp.so (include/sgp.h).  One native context per executor task; device = partitionId % nGPUs. */
/** What the JNI glue throws for every non-zero status of the C-ABI: message = "SGP<code>: <sgp_last_error>". */
class SgpNativeException(message: String) extends RuntimeException(message) {
  def code: Int = message.drop(3).takeWhile(_.isDigit).toInt
}

private[ml] object NativeProjectedProcess {
  System.loadLibrary("sgp_jni")
  @native def create(device: Int): Long
  @native def destroy(ctx: Long): Unit
  @native def begin(ctx: Long, types: Array[Int], scales: Array[Double], sigmas: Array[Double], betas: Array[Double],
                    activeSet: Array[Double], m: Int, d: Int): Unit
  @native def accumulate(ctx: Long, x: Array[Double], y: Array[Double], n: Long): Unit
  @native def finish(ctx: Long, g: Array[Double], b: Array[Double]): Unit
  @native def magic(ctx: Long, g: Array[Double], b: Array[Double], magicVector: Array[Double],
                    magicMatrix: Array[Double]): Unit
  /** Installs (magicVector, magicMatrix) for predict; the matrix may be Breeze's column-major array (same quadratic form). */
  @native def setMagic(ctx: Long, magicVector: Array[Double], magicMatrix: Array[Double]): Unit
  /** mean (and var, unless null) of n rows of x (row-major): GaussianProjectedProcessRawPredictor.predict, GPC:121-125. */
  @native def predict(ctx: Long, x: Array[Double], n: Long, mean: Array[Double], variance: Array[Double]): Unit
  /** p (and mean, variance, unless null) of n rows of x (row-major): the probability of class 1 averaged over the latent
    * posterior, new Integrator(nodes).expectedOfFunctionOfNormal(mean, variance, sigmoid) on the device, a negative
    * variance taken as 0 (commons/util/Integrator.scala; IntegratorTest uses nodes = 100). */
  @native def predictProbability(ctx: Long, x: Array[Double], n: Long, nodes: Int, p: Array[Double], mean: Array[Double],
                                 variance: Array[Double]): Unit

  /** The averaged probability of class 1 for one partition's rows under a binary classification model (kernel,
    * activeSet, magicVector, magicMatrix), in blocks of `block` rows: what `scorePartition` is for the raw prediction. */
  def probabilityPartition(partitionId: Int, rows: Iterator[Vector], kernel: Kernel, activeSet: Array[Vector],
                           magicVector: BDV[Double], magicMatrix: BDM[Double], nodes: Int = 100,
                           nGPUs: Int = 8, block: Int = 32768): Iterator[Double] = {
    val m = activeSet.length
    val d = activeSet.head.size
    val terms = flatten(kernel)
    val ctx = create(partitionId % nGPUs)
    try {
      begin(ctx, terms.map(_._1).toArray, terms.map(_._2).toArray, terms.map(_._3).toArray, terms.flatMap(_._4).toArray,
        activeSet.flatMap(_.toArray), m, d)
      setMagic(ctx, magicVector.toArray, magicMatrix.toArray)
      rows.grouped(block).flatMap { blk =>
        val p = new Array[Double](blk.length)
        predictProbability(ctx, blk.flatMap(_.toArray).toArray, blk.length.toLong, nodes, p, null, null)
        p.iterator
      }.toVector.iterator                                   // materialised: the context is destroyed below
    } finally destroy(ctx)
  }

  /** Scores one partition's rows with the model (kernel, activeSet, magicVector, magicMatrix): one native context per
    * task (device = partitionId % nGPUs), rows in blocks of `block`.  What a model's `transform` maps over its partitions
    * (`dataset.rdd.mapPartitionsWithIndex`), instead of one Breeze row at a time (GPC:121-125). */
  def scorePartition(partitionId: Int, rows: Iterator[Vector], kernel: Kernel, activeSet: Array[Vector],
                     magicVector: BDV[Double], magicMatrix: BDM[Double], withVariance: Boolean,
                     nGPUs: Int = 8, block: Int = 32768): Iterator[(Double, Double)] = {
    val m = activeSet.length
    val d = activeSet.head.size
    val terms = flatten(kernel)
    val ctx = create(partitionId % nGPUs)
    try {
      begin(ctx, terms.map(_._1).toArray, terms.map(_._2).toArray, terms.map(_._3).toArray, terms.flatMap(_._4).toArray,
        activeSet.flatMap(_.toArray), m, d)
      setMagic(ctx, magicVector.toArray, magicMatrix.toArray)
      rows.grouped(block).flatMap { blk =>
        val n = blk.length
        val mean = new Array[Double](n)
        val variance = if (withVariance) new Array[Double](n) else null
        predict(ctx, blk.flatMap(_.toArray).toArray, n.toLong, mean, variance)
        mean.indices.iterator.map(i => (mean(i), if (withVariance) variance(i) else Double.NaN))
      }.toVector.iterator                                   // materialised: the context is destroyed below
    } finally destroy(ctx)
  }
  // hyper-parameter objective: experts resident on the GPU, one native call per objective evaluation
  @native def expertsUpload(ctx: Long, x: Array[Double], y: Array[Double], offsets: Array[Long], d: Int): Unit
  /** [value, gradient...]; tol <= 0: regression NLL (GPR:55-68), tol > 0: the classifier's Laplace objective. */
  @native def objective(ctx: Long, types: Array[Int], scales: Array[Double], sigmas: Array[Double], betas: Array[Double],
                        d: Int, hKind: Array[Int], hTerm: Array[Int], hDim: Array[Int], hValue: Array[Double],
                        hCoef: Array[Double], tol: Double): Array[Double]
  @native def expertsGetF(ctx: Long, f: Array[Double]): Unit
  /** Row indices of the points GreedilyOptimizingActiveSetProvider selects (ActiveSetProvider.scala:58-139) among the n
    * points of x (row-major, d columns); rank-1 updates on the device.  firstIndex replaces takeSample(1, seed), ASP:70;
    * nExperts = Math.round(n / datasetSizeForExpert), GPC:27. */
  @native def greedyActiveSet(ctx: Long, types: Array[Int], scales: Array[Double], sigmas: Array[Double],
                              betas: Array[Double], x: Array[Double], y: Array[Double], n: Long, d: Int, nExperts: Long,
                              firstIndex: Long, activeSetSize: Int): Array[Long]
  /** Centres (k_out x d row-major) of Spark 3.1 MLlib KMeans with the reference's settings (k-means||, tol 1e-4) over the
    * n points of x (row-major, d columns), computed on the device (sgp_kmeans). */
  @native def kmeansActiveSet(ctx: Long, x: Array[Double], n: Long, d: Int, k: Int, maxIter: Int, seed: Long): Array[Double]

  /** Flattens the kernel DSL tree into (type, scale, sigma, beta) terms; `scale` multiplies down the tree
    * (ScalarTimesKernel.scala:20-28), Eye terms are kept (they carry whiteNoiseVar / the K_mm diagonal). */
  def flatten(k: Kernel, scale: Double = 1d): Seq[(Int, Double, Double, Array[Double])] = k match {
    case s: SumOfKernels       => flatten(s.kernel1, scale) ++ flatten(s.kernel2, scale)   // needs the two vals exposed
    case c: ScalarTimesKernel  => flatten(c.innerKernel, scale * c.scalar)                 // ditto (kernel, C)
    case a: ARDRBFKernel       => Seq((0, scale, 0d, a.getHyperparameters.toArray))
    case r: RBFKernel          => Seq((1, scale, r.getHyperparameters(0), Array.empty[Double]))
    case _: EyeKernel          => Seq((2, scale, 0d, Array.empty[Double]))
  }

  /** One descriptor per hyper-parameter, in `getHyperparameters` order (depth first, a trainable scalar PREPENDED to
    * its inner kernel's vector, ScalarTimesKernel.scala:76-82), saying how the kernel matrix depends on it:
    * (kind, term, dim, value, coef) with kind 0 = trainable scalar (coef(t) = d scale_t / d theta for every flattened
    * term t, i.e. the scale of the inner term WITHOUT this C, ScalarTimesKernel.scala:93-97), 1 = ARD beta_k of term t
    * (ARDRBFKernel.scala:61-79), 2 = RBF sigma of term t (RBFKernel.scala:56-64).  `offset` = index of the first
    * flattened term of this sub-tree. */
  case class Hyper(kind: Int, term: Int, dim: Int, value: Double, coef: Map[Int, Double])
  def describe(k: Kernel, scale: Double = 1d, offset: Int = 0): Seq[Hyper] = k match {
    case s: SumOfKernels =>
      describe(s.kernel1, scale, offset) ++ describe(s.kernel2, scale, offset + flatten(s.kernel1).length)
    case t: TrainableScalarTimesKernel =>
      val inner = flatten(t.innerKernel, scale)
      Hyper(0, 0, 0, t.scalar, inner.zipWithIndex.map { case (term, i) => (offset + i) -> term._2 }.toMap) +:
        describe(t.innerKernel, scale * t.scalar, offset)
    case c: ScalarTimesKernel => describe(c.innerKernel, scale * c.scalar, offset)
    case a: ARDRBFKernel      => a.getHyperparameters.toArray.zipWithIndex.map { case (b, j) => Hyper(1, offset, j, b, Map.empty) }
    case r: RBFKernel         => Seq(Hyper(2, offset, 0, r.getHyperparameters(0), Map.empty))
    case _: EyeKernel         => Seq.empty
  }

  /** One objective evaluation on an executor's resident experts (the body of the treeAggregate in
    * GaussianProcessCommons.scala:73-78): returns (value, gradient). */
  def evaluate(ctx: Long, kernel: Kernel, d: Int, tol: Double): (Double, BDV[Double]) = {
    val terms = flatten(kernel)
    val hs = describe(kernel)
    val coef = hs.flatMap(h => terms.indices.map(t => h.coef.getOrElse(t, 0d))).toArray      // [h][n_terms]
    val out = objective(ctx, terms.map(_._1).toArray, terms.map(_._2).toArray, terms.map(_._3).toArray,
      terms.flatMap(_._4).toArray, d, hs.map(_.kind).toArray, hs.map(_.term).toArray, hs.map(_.dim).toArray,
      hs.map(_.value).toArray, coef, tol)
    (out(0), new BDV(out.drop(1)))
  }
}

/** Drop-in for KMeansActiveSetProvider (ActiveSetProvider.scala:22-46): the points are collected to the driver and
  * clustered on its GPU in one native call instead of Spark MLlib's distributed KMeans (same algorithm and settings;
  * Spark's partition-dependent RNG streams are replaced by the library's counter-based generator). */
class NativeKMeansActiveSetProvider(private val maxIter: Int = 20, device: Int = 0) extends ActiveSetProvider {
  override def apply(activeSetSize: Int,
                     expertLabelsAndKernels: RDD[(BDV[Double], Kernel)],
                     points: RDD[org.apache.spark.ml.feature.LabeledPoint],
                     kernel: () => Kernel,
                     optimalHyperparameter: BDV[Double],
                     seed: Long): Array[Vector] = {
    val rows = points.map(_.features.toArray).collect()
    val d = rows.head.length
    val ctx = NativeProjectedProcess.create(device)
    try {
      val c = NativeProjectedProcess.kmeansActiveSet(ctx, rows.flatten, rows.length.toLong, d, activeSetSize, maxIter, seed)
      c.grouped(d).map(r => org.apache.spark.ml.linalg.Vectors.dense(r): Vector).toArray
    } finally NativeProjectedProcess.destroy(ctx)
  }
}

/** Drop-in for ProjectedGaussianProcessHelper (commons/ProjectedGaussianProcessHelper.scala): same two methods,
  * same return types; mix this trait into GaussianProcessCommons instead of the original. */
private[ml] trait NativeProjectedGaussianProcessHelper extends ProjectedGaussianProcessHelper {
  /** Status codes of include/sgp.h back to the reference's exception types (the inner class NotPositiveDefiniteException,
    * PGPH:9-11, needs this trait instance as its outer object, which is why the mapping lives here and not in the JNI). */
  protected def rethrow[T](body: => T): T =
    try body catch {
      case e: SgpNativeException => e.code match {
        case 3 => throw new NotPositiveDefiniteException                                           // SGP_E_NOT_PD
        case 1 => throw new IllegalArgumentException(e.getMessage)                                  // SGP_E_BADARG
        case 5 => throw new org.apache.spark.ml.commons.kernel.TrainingVectorsNotInitializedException  // SGP_E_STATE
        case 6 => throw new breeze.linalg.MatrixSingularException(e.getMessage)                     // SGP_E_SINGULAR
        case _ => throw e
      }
    }

  import NativeProjectedProcess._

  def nGPUs: Int = 8

  override def getMatrixKmnKnmAndVectorKmny(expertLabelsAndKernels: RDD[(BDV[Double], Kernel)],
                                            activeSet: Array[Vector]): (BDM[Double], BDV[Double]) = {
    val m = activeSet.length
    val d = activeSet.head.size
    val z = activeSet.flatMap(_.toArray)
    val terms = flatten(expertLabelsAndKernels.first()._2)        // every expert carries the same kernel / theta
    val (ty, sc, sg, be) = (terms.map(_._1).toArray, terms.map(_._2).toArray, terms.map(_._3).toArray,
      terms.flatMap(_._4).toArray)
    // seqOp of PGPH:25-30 becomes: one native context per partition, all experts of the partition in one shard
    val partials = expertLabelsAndKernels.mapPartitionsWithIndex { (pid, it) =>
      val ctx = create(pid % nGPUs)
      try {
        begin(ctx, ty, sc, sg, be, z, m, d)
        it.grouped(256).foreach { experts =>                      // pack a few hundred experts per native call
          val x = experts.flatMap(_._2.getTrainingVectors.flatMap(_.toArray)).toArray
          val y = experts.flatMap(_._1.toArray).toArray
          accumulate(ctx, x, y, y.length.toLong)
        }
        val g = new Array[Double](m * m); val b = new Array[Double](m)
        finish(ctx, g, b)
        Iterator.single((new BDM(m, m, g), new BDV(b)))
      } finally destroy(ctx)
    }
    partials.treeReduce { case ((g1, b1), (g2, b2)) => (g1 += g2, b1 += b2) }   // combOp, PGPH:31-35
  }

  override def getMagicVector(kernel: Kernel, matrixKmnKnm: BDM[Double], vectorKmny: BDV[Double],
                              activeSet: Array[Vector], optimalHyperparameter: BDV[Double]) = {
    val m = activeSet.length
    val d = activeSet.head.size
    val terms = flatten(kernel)
    val ctx = create(0)
    try {
      begin(ctx, terms.map(_._1).toArray, terms.map(_._2).toArray, terms.map(_._3).toArray,
        terms.flatMap(_._4).toArray, activeSet.flatMap(_.toArray), m, d)
      val mv = new Array[Double](m); val mm = new Array[Double](m * m)
      rethrow(magic(ctx, matrixKmnKnm.toArray, vectorKmny.toArray, mv, mm))   // NotPositiveDefiniteException like PGPH:62-65
      (new BDV(mv), new BDM(m, m, mm))
    } finally destroy(ctx)
  }
}
