/*
 * native-als: what the engine templates call instead of org.apache.spark.mllib.recommendation.ALS.
 *
 * Same parameters as the MLlib calls it displaces
 *   new ALS().setRank(..)...run(ratings)   examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:76-86
 *   ALS.train(ratings, rank, iterations, lambda, -1, seed)
 *                                           examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/ECommAlgorithm.scala:116-122
 *   ALS.trainImplicit(ratings, rank, iterations, lambda, -1, 1.0, seed)
 *                                           examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:121-128
 * and the same result fields the templates read (rank, userFeatures, productFeatures, recommendProducts).
 * All arithmetic happens in libpio_als.so (CUDA, sm_90a) behind the JNI shim src/main/c/pio_als_jni.c; this file only
 * collects the ratings to primitive arrays and owns the native handle.
 */
package org.apache.predictionio.nativeals

import org.apache.spark.mllib.recommendation.Rating
import org.apache.spark.rdd.RDD

object NativeALS {
  System.loadLibrary("pio_als_jni") // links libpio_als.so (java.library.path / LD_LIBRARY_PATH)

  // ---- natives: one per entry point of include/pio_als.h (pio_als_jni.c) ----------------------------------
  @native def create(rank: Int, implicitPrefs: Boolean, nUsers: Int, nItems: Int, lambda: Double, alpha: Double,
    seed: Long, device: Int, worldSize: Int, worldRank: Int, ncclId: Array[Byte]): Long
  @native def destroy(h: Long): Unit
  @native def ncclUniqueId(): Array[Byte]
  @native def setRatings(h: Long, user: Array[Int], item: Array[Int], rating: Array[Float], dedup: Int,
    ts: Array[Long]): Unit
  @native def setInit(h: Long, userFactors: Array[Float], itemFactors: Array[Float]): Unit
  @native def run(h: Long, iterations: Int): Unit
  @native def getFactors(h: Long, userOut: Array[Float], itemOut: Array[Float], userHas: Array[Byte],
    itemHas: Array[Byte]): Unit
  @native def train(h: Long, user: Array[Int], item: Array[Int], rating: Array[Float], dedup: Int, ts: Array[Long],
    userInit: Array[Float], itemInit: Array[Float], iterations: Int, userOut: Array[Float], itemOut: Array[Float],
    userHas: Array[Byte], itemHas: Array[Byte]): Unit
  @native def recommend(h: Long, users: Array[Int], topk: Int, itemMask: Array[Byte], itemWeight: Array[Double],
    outItems: Array[Int], outScores: Array[Float], outCount: Array[Int]): Unit
  @native def similar(h: Long, queryItems: Array[Int], topk: Int, itemMask: Array[Byte], itemWeight: Array[Double],
    flags: Int, outItems: Array[Int], outScores: Array[Float]): Int
  @native def similarBatch(h: Long, queryPtr: Array[Long], queryItems: Array[Int], topk: Int, itemMask: Array[Byte],
    itemWeight: Array[Double], flags: Int, outItems: Array[Int], outScores: Array[Float], outCount: Array[Int]): Unit
  /** recommend / similarBatch with a filter per query (pio_als_query_filter as arrays, any of them null): exclusion
    * lists (exPtr / exItems), white lists (hasWl / wlPtr / wlItems) and shared set rows (setIx into itemSets). */
  @native def recommendFiltered(h: Long, users: Array[Int], topk: Int, itemMask: Array[Byte], itemWeight: Array[Double],
    exPtr: Array[Long], exItems: Array[Int], hasWl: Array[Byte], wlPtr: Array[Long], wlItems: Array[Int],
    setIx: Array[Int], itemSets: Array[Byte], nSets: Int, outItems: Array[Int], outScores: Array[Float],
    outCount: Array[Int]): Unit
  @native def similarBatchFiltered(h: Long, queryPtr: Array[Long], queryItems: Array[Int], topk: Int,
    itemMask: Array[Byte], itemWeight: Array[Double], flags: Int, exPtr: Array[Long], exItems: Array[Int],
    hasWl: Array[Byte], wlPtr: Array[Long], wlItems: Array[Int], setIx: Array[Int], itemSets: Array[Byte], nSets: Int,
    outItems: Array[Int], outScores: Array[Float], outCount: Array[Int]): Unit
  @native def save(h: Long, path: String): Unit
  @native def load(path: String, device: Int): Long
  @native def importModel(rank: Int, nUsers: Int, nItems: Int, device: Int, userFactors: Array[Float],
    itemFactors: Array[Float], userHas: Array[Byte], itemHas: Array[Byte]): Long
  @native def stats(h: Long): Array[Long]
  @native def nbTrain(device: Int, label: Array[Int], x: Array[Float], nFeat: Int, nClass: Int,
    lambda: Double): Array[Double]
  @native def encodeIds(device: Int, bytes: Array[Byte], offsets: Array[Long], outFirst: Array[Long]): Array[Int]
  @native def coocTrain(device: Int, user: Array[Int], item: Array[Int], nUsers: Int, nItems: Int, topn: Int,
    outItem: Array[Int], outCount: Array[Int], outN: Array[Int]): Unit

  /** BiMap.stringInt(keys) on the device (BiMap.scala:116-128): index per key in first-occurrence order and the keys of
    * the distinct ids in index order. */
  def stringInt(keys: Array[String], device: Int = 0): (Array[Int], Array[String]) = {
    val enc = keys.map(_.getBytes("UTF-8"))
    val offsets = enc.scanLeft(0L)(_ + _.length)
    val first = new Array[Long](keys.length)
    val idx = encodeIds(device, enc.flatten, offsets, first)
    val n = if (idx.isEmpty) 0 else idx.max + 1
    (idx, first.take(n).map(p => keys(p.toInt)))
  }

  /** How repeated (user, item) pairs are treated (the templates' own reduceByKey, moved to the device). */
  val DEDUP_NONE = 0      // recommendation: every event is its own rating (ALSAlgorithm.scala:62-65)
  val DEDUP_SUM = 1       // similarproduct: reduceByKey(_ + _) (multi-events ALSAlgorithm.scala:106)
  val DEDUP_KEEP_LAST = 2 // ecommerce: latest timestamp wins (ECommAlgorithm.scala:189-197)
  /** pio_als_similar flag: query items stay candidates (ecommerce predictSimilar, ECommAlgorithm.scala:492-525). */
  val SIM_KEEP_QUERY_ITEMS = 1

  /** Drop-in for `new ALS()....run(ratings)` / `ALS.train` / `ALS.trainImplicit`.
    * nUsers / nItems are the sizes of the templates' BiMaps (indices are 0 until n). */
  def run(ratings: RDD[Rating], nUsers: Int, nItems: Int, rank: Int, iterations: Int, lambda: Double,
    implicitPrefs: Boolean, alpha: Double, seed: Long, dedup: Int = DEDUP_NONE,
    times: Option[RDD[Long]] = None, device: Int = 0): NativeModel = {
    require(!ratings.take(1).isEmpty, "ratings cannot be empty.")
    val rs = ratings.map(r => (r.user, r.product, r.rating.toFloat)).collect()
    val ts = times.map(_.collect()).orNull
    val h = create(rank, implicitPrefs, nUsers, nItems, lambda, alpha, seed, device, 1, 0, null)
    try {
      val uf = new Array[Float](nUsers * rank)
      val pf = new Array[Float](nItems * rank)
      val uh = new Array[Byte](nUsers)
      val ph = new Array[Byte](nItems)
      train(h, rs.map(_._1), rs.map(_._2), rs.map(_._3), dedup, ts, null, null, iterations, uf, pf, uh, ph)
      new NativeModel(h, rank, nUsers, nItems, uf, pf, uh, ph)
    } catch {
      case e: Throwable => destroy(h); throw e
    }
  }

  def train(ratings: RDD[Rating], nUsers: Int, nItems: Int, rank: Int, iterations: Int, lambda: Double,
    seed: Long): NativeModel =
    run(ratings, nUsers, nItems, rank, iterations, lambda, implicitPrefs = false, alpha = 1.0, seed = seed)

  def trainImplicit(ratings: RDD[Rating], nUsers: Int, nItems: Int, rank: Int, iterations: Int, lambda: Double,
    alpha: Double, seed: Long): NativeModel =
    run(ratings, nUsers, nItems, rank, iterations, lambda, implicitPrefs = true, alpha = alpha, seed = seed)
}

/** The trained model: the native handle (device-resident factors, used for scoring) plus host copies of the factors in
  * the shape MatrixFactorizationModel exposes.  Rows whose `has` flag is 0 never occurred in the ratings: MLlib emits
  * no factor for them, here they are zero rows that the scoring entry points skip. */
class NativeModel(
  @transient private var handle: Long,
  val rank: Int,
  val nUsers: Int,
  val nItems: Int,
  val userFactors: Array[Float],
  val productFactors: Array[Float],
  val userHas: Array[Byte],
  val productHas: Array[Byte]) extends Serializable {

  private def h: Long = {
    if (handle == 0L) {
      // after Kryo / Java deserialisation on another JVM: rebuild the device copy from the host factors
      handle = NativeALS.importModel(rank, nUsers, nItems, 0, userFactors, productFactors, userHas, productHas)
    }
    handle
  }

  /** MatrixFactorizationModel.userFeatures / productFeatures as the templates collect them. */
  def userFeatures: Iterator[(Int, Array[Double])] = rows(userFactors, userHas)
  def productFeatures: Iterator[(Int, Array[Double])] = rows(productFactors, productHas)
  private def rows(f: Array[Float], has: Array[Byte]): Iterator[(Int, Array[Double])] =
    has.indices.iterator.filter(has(_) != 0).map(i => (i, f.slice(i * rank, (i + 1) * rank).map(_.toDouble)))

  /** recommendProducts / recommendProductsWithFilter (ALSModel.scala:44-60): best `num` items per user, blacklist as a
    * byte mask over the item indices; batch form = batchPredict (ALSAlgorithm.scala:117-158). */
  def recommendProducts(users: Array[Int], num: Int, itemMask: Array[Byte] = null,
    itemWeight: Array[Double] = null): Array[Array[(Int, Double)]] = {
    val oi = new Array[Int](users.length * num)
    val os = new Array[Float](users.length * num)
    val oc = new Array[Int](users.length)
    NativeALS.recommend(h, users, num, itemMask, itemWeight, oi, os, oc)
    users.indices.map(q => (0 until oc(q)).map(t => (oi(q * num + t), os(q * num + t).toDouble)).toArray).toArray
  }

  /** similarproduct predict: sum of cosines against the query items, score > 0 only (ALSAlgorithm.scala:138-197). */
  def similarProducts(queryItems: Array[Int], num: Int, itemMask: Array[Byte] = null,
    itemWeight: Array[Double] = null, keepQueryItems: Boolean = false): Array[(Int, Double)] = {
    val oi = new Array[Int](num)
    val os = new Array[Float](num)
    val n = NativeALS.similar(h, queryItems, num, itemMask, itemWeight,
      if (keepQueryItems) NativeALS.SIM_KEEP_QUERY_ITEMS else 0, oi, os)
    (0 until n).map(t => (oi(t), os(t).toDouble)).toArray
  }

  def save(path: String): Unit = NativeALS.save(h, path)
  def close(): Unit = if (handle != 0L) { NativeALS.destroy(handle); handle = 0L }
  override def finalize(): Unit = close()
}

object NativeModel {
  def load(path: String, rank: Int, nUsers: Int, nItems: Int, device: Int = 0): NativeModel = {
    val hd = NativeALS.load(path, device)
    val uf = new Array[Float](nUsers * rank)
    val pf = new Array[Float](nItems * rank)
    val uh = new Array[Byte](nUsers)
    val ph = new Array[Byte](nItems)
    NativeALS.getFactors(hd, uf, pf, uh, ph)
    new NativeModel(hd, rank, nUsers, nItems, uf, pf, uh, ph)
  }
}
