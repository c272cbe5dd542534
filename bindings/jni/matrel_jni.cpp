// JNI shim between the Scala facade (bindings/scala/Dataset.scala) and the C ABI (include/matrel.h).
// NOT compiled in this image (no JDK: `javac`, `jni.h` absent); it is the binding a maintainer adds:
//   g++ -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude bindings/jni/matrel_jni.cpp \
//       -Lmatrel_b200 -lmatrel_b200 -o libmatrel_jni.so
// tests/test_abi_cpu.py type-checks it against include/matrel.h with a stand-in <jni.h> (tests/cpp/jni_stub).
//
// Array traffic uses Get/Set<Type>ArrayRegion into native staging vectors, never GetPrimitiveArrayCritical: the ABI calls
// allocate device memory, take locks and may wait on streams, none of which is allowed inside a JNI critical region.
// Staging memory is pageable, so cudaMemcpyAsync has consumed it when mr_matrix_put_block returns.
#if __has_include(<jni.h>)
#include <jni.h>

#include <cstdint>
#include <vector>

#include "matrel.h"

namespace {
// `require` failures become IllegalArgumentException with the reference's message text.
bool throw_if(JNIEnv* env, mr_status st) {
  if (st == MR_OK) return false;
  const char* cls = (st == MR_EINVAL || st == MR_EDIM) ? "java/lang/IllegalArgumentException"
                    : (st == MR_ENOMEM)                ? "java/lang/OutOfMemoryError"
                    : (st == MR_ENOTSUP)               ? "java/lang/UnsupportedOperationException"
                    : (st == MR_ENOTFOUND)             ? "java/util/NoSuchElementException"
                                                       : "java/lang/RuntimeException";  // MR_ECUDA, MR_ENCCL
  jclass c = env->FindClass(cls);
  if (c != nullptr) env->ThrowNew(c, mr_last_error());
  return true;
}
bool throw_iae(JNIEnv* env, const char* msg) {
  jclass c = env->FindClass("java/lang/IllegalArgumentException");
  if (c != nullptr) env->ThrowNew(c, msg);
  return true;
}
template <typename T>
T* ptr(jlong h) { return reinterpret_cast<T*>(static_cast<intptr_t>(h)); }

// The 7 fields of MLMatrixSerializer.serialize (util/MLMatrixSerializer.scala:26-48) staged in native memory.
struct StagedBlock {
  mr_block_desc d{};
  std::vector<double> values;
  std::vector<int32_t> colPtrs, rowIndices;
  bool ok = false;
  StagedBlock(JNIEnv* env, jbyte type, jint numRows, jint numCols, jintArray jcolPtrs, jintArray jrowIndices, jdoubleArray jvalues,
              jboolean isTransposed) {
    if (jvalues == nullptr) {
      throw_iae(env, "requirement failed: values is null");
      return;
    }
    if (type == 0 && (jcolPtrs == nullptr || jrowIndices == nullptr)) {
      throw_iae(env, "requirement failed: colPtrs / rowIndices is null for a SparseMatrix");
      return;
    }
    values.resize(static_cast<size_t>(env->GetArrayLength(jvalues)));
    if (!values.empty()) env->GetDoubleArrayRegion(jvalues, 0, static_cast<jsize>(values.size()), values.data());
    if (type == 0) {
      colPtrs.resize(static_cast<size_t>(env->GetArrayLength(jcolPtrs)));
      rowIndices.resize(static_cast<size_t>(env->GetArrayLength(jrowIndices)));
      if (!colPtrs.empty()) env->GetIntArrayRegion(jcolPtrs, 0, static_cast<jsize>(colPtrs.size()), colPtrs.data());
      if (!rowIndices.empty()) env->GetIntArrayRegion(jrowIndices, 0, static_cast<jsize>(rowIndices.size()), rowIndices.data());
    }
    if (env->ExceptionCheck()) return;
    d.type = static_cast<uint8_t>(type);
    d.numRows = numRows;
    d.numCols = numCols;
    d.isTransposed = isTransposed ? 1 : 0;
    d.values = values.data();
    d.valuesLen = static_cast<int64_t>(values.size());
    if (type == 0) {
      d.colPtrs = colPtrs.data();
      d.colPtrsLen = static_cast<int64_t>(colPtrs.size());
      d.rowIndices = rowIndices.data();
      d.rowIndicesLen = static_cast<int64_t>(rowIndices.size());
    }
    ok = true;
  }
};

// {type, numRows, numCols, isTransposed, valuesLen, colPtrsLen, rowIndicesLen} of a block (first call of the two-call protocol)
jlongArray meta_of(JNIEnv* env, const mr_block_desc& d) {
  const jlong f[7] = {d.type, d.numRows, d.numCols, d.isTransposed, d.valuesLen, d.colPtrsLen, d.rowIndicesLen};
  jlongArray out = env->NewLongArray(7);
  if (out != nullptr) env->SetLongArrayRegion(out, 0, 7, f);
  return out;
}
// second call: the arrays, copied into JVM arrays of the lengths meta_of reported
template <typename Get>
void arrays_into(JNIEnv* env, Get&& get, jintArray jcolPtrs, jintArray jrowIndices, jdoubleArray jvalues) {
  mr_block_desc d{};
  if (throw_if(env, get(&d))) return;  // sizes
  std::vector<double> values(static_cast<size_t>(d.valuesLen));
  std::vector<int32_t> colPtrs(static_cast<size_t>(d.colPtrsLen)), rowIndices(static_cast<size_t>(d.rowIndicesLen));
  if (jvalues == nullptr || env->GetArrayLength(jvalues) < d.valuesLen ||
      (d.type == 0 && (jcolPtrs == nullptr || jrowIndices == nullptr || env->GetArrayLength(jcolPtrs) < d.colPtrsLen ||
                       env->GetArrayLength(jrowIndices) < d.rowIndicesLen))) {
    throw_iae(env, "requirement failed: destination arrays are null or too short");
    return;
  }
  d.values = values.data();
  d.colPtrs = d.type == 0 ? colPtrs.data() : nullptr;
  d.rowIndices = d.type == 0 ? rowIndices.data() : nullptr;
  if (throw_if(env, get(&d))) return;
  if (!values.empty()) env->SetDoubleArrayRegion(jvalues, 0, static_cast<jsize>(values.size()), values.data());
  if (d.type == 0) {
    if (!colPtrs.empty()) env->SetIntArrayRegion(jcolPtrs, 0, static_cast<jsize>(colPtrs.size()), colPtrs.data());
    if (!rowIndices.empty()) env->SetIntArrayRegion(jrowIndices, 0, static_cast<jsize>(rowIndices.size()), rowIndices.data());
  }
}
}  // namespace

#define MR_JNI(RET, NAME) JNIEXPORT RET JNICALL Java_org_apache_spark_sql_matfast_b200_Native_##NAME

extern "C" {

// ---- session: MatfastSession.builder().getOrCreate() (MatfastSession.scala:177-234)
MR_JNI(jlong, init)(JNIEnv* env, jclass, jint device, jboolean compat, jint gemmAlgo) {
  mr_options o{};
  o.device = device;
  o.compat_bugs = compat ? 1 : 0;
  o.gemm_algo = gemmAlgo;
  mr_context* ctx = nullptr;
  if (throw_if(env, mr_init(&o, &ctx))) return 0;
  return reinterpret_cast<jlong>(ctx);
}
MR_JNI(void, shutdown)(JNIEnv* env, jclass, jlong ctx) { throw_if(env, mr_shutdown(ptr<mr_context>(ctx))); }
MR_JNI(void, sync)(JNIEnv* env, jclass, jlong ctx) { throw_if(env, mr_sync(ptr<mr_context>(ctx))); }

// ---- datasets: Seq(MatrixBlock(...)).toDS() and .collect()
MR_JNI(jlong, matrixCreate)(JNIEnv* env, jclass, jlong ctx) {
  mr_matrix* m = nullptr;
  if (throw_if(env, mr_matrix_create(ptr<mr_context>(ctx), &m))) return 0;
  return reinterpret_cast<jlong>(m);
}
MR_JNI(void, matrixFree)(JNIEnv* env, jclass, jlong m) { throw_if(env, mr_matrix_free(ptr<mr_matrix>(m))); }
// host-resident datasets: put_block copies the JVM arrays into page-locked memory owned by the library, so the staged
// arrays are released as soon as the call returns
MR_JNI(jlong, matrixCreateHost)(JNIEnv* env, jclass, jlong ctx) {
  mr_matrix* m = nullptr;
  if (throw_if(env, mr_matrix_create_host(ptr<mr_context>(ctx), &m))) return 0;
  return reinterpret_cast<jlong>(m);
}
MR_JNI(jboolean, isHost)(JNIEnv* env, jclass, jlong m) {
  int32_t host = 0;
  throw_if(env, mr_matrix_is_host(ptr<mr_matrix>(m), &host));
  return host != 0;
}
MR_JNI(jlong, toHost)(JNIEnv* env, jclass, jlong m) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_matrix_to_host(ptr<mr_matrix>(m), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, toDevice)(JNIEnv* env, jclass, jlong m) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_matrix_to_device(ptr<mr_matrix>(m), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
// a whole matrix: `values` column-major (DenseMatrix.values of an nrows x ncols matrix), staged in pageable native memory, so it is
// free again when mr_matrix_from_dense returns
MR_JNI(jlong, matrixFromArray)(JNIEnv* env, jclass, jlong ctx, jdoubleArray jvalues, jlong nrows, jlong ncols, jint blkSize) {
  if (jvalues == nullptr || nrows <= 0 || ncols <= 0 || env->GetArrayLength(jvalues) != nrows * ncols) {
    throw_iae(env, "requirement failed: values must hold nrows * ncols elements");
    return 0;
  }
  std::vector<double> values(static_cast<size_t>(nrows * ncols));
  env->GetDoubleArrayRegion(jvalues, 0, static_cast<jsize>(values.size()), values.data());
  if (env->ExceptionCheck()) return 0;
  mr_matrix* m = nullptr;
  if (throw_if(env, mr_matrix_from_dense(ptr<mr_context>(ctx), values.data(), nrows, ncols, nrows, 0, blkSize, 0, nullptr, &m))) return 0;
  return reinterpret_cast<jlong>(m);
}
// DenseMatrix.toArray for the whole dataset into `out` (column-major, nrows * ncols elements, allocated by the caller)
MR_JNI(void, matrixToArray)(JNIEnv* env, jclass, jlong m, jlong nrows, jlong ncols, jint blkSize, jdoubleArray out) {
  if (out == nullptr || nrows <= 0 || ncols <= 0 || env->GetArrayLength(out) != nrows * ncols) {
    throw_iae(env, "requirement failed: the destination must hold nrows * ncols elements");
    return;
  }
  std::vector<double> values(static_cast<size_t>(nrows * ncols));
  if (throw_if(env, mr_matrix_to_dense(ptr<mr_matrix>(m), nrows, ncols, blkSize, values.data(), nrows, 0, nullptr))) return;
  env->SetDoubleArrayRegion(out, 0, static_cast<jsize>(values.size()), values.data());
}
MR_JNI(void, putBlock)(JNIEnv* env, jclass, jlong m, jint rid, jint cid, jbyte type, jint numRows, jint numCols, jintArray colPtrs,
                       jintArray rowIndices, jdoubleArray values, jboolean isTransposed) {
  StagedBlock b(env, type, numRows, numCols, colPtrs, rowIndices, values, isTransposed);
  if (!b.ok) return;
  throw_if(env, mr_matrix_put_block(ptr<mr_matrix>(m), rid, cid, &b.d));
}
MR_JNI(jlong, numBlocks)(JNIEnv* env, jclass, jlong m) {
  int64_t n = 0;
  throw_if(env, mr_matrix_num_blocks(ptr<mr_matrix>(m), &n));
  return n;
}
MR_JNI(jboolean, hasBlock)(JNIEnv* env, jclass, jlong m, jint rid, jint cid) {
  int32_t has = 0;
  throw_if(env, mr_matrix_has_block(ptr<mr_matrix>(m), rid, cid, &has));
  return has != 0;
}
// (rid_0, cid_0, rid_1, cid_1, ...) in ascending (rid, cid) order
MR_JNI(jintArray, blockIds)(JNIEnv* env, jclass, jlong m) {
  int64_t n = 0;
  if (throw_if(env, mr_matrix_num_blocks(ptr<mr_matrix>(m), &n))) return nullptr;
  std::vector<int32_t> rids(static_cast<size_t>(n)), cids(static_cast<size_t>(n)), both(static_cast<size_t>(2 * n));
  if (n > 0 && throw_if(env, mr_matrix_block_ids(ptr<mr_matrix>(m), rids.data(), cids.data(), n))) return nullptr;
  for (int64_t i = 0; i < n; ++i) {
    both[static_cast<size_t>(2 * i)] = rids[static_cast<size_t>(i)];
    both[static_cast<size_t>(2 * i + 1)] = cids[static_cast<size_t>(i)];
  }
  jintArray out = env->NewIntArray(static_cast<jsize>(2 * n));
  if (out != nullptr && n > 0) env->SetIntArrayRegion(out, 0, static_cast<jsize>(2 * n), both.data());
  return out;
}
// MLMatrixSerializer.serialize, two calls: blockMeta sizes the JVM arrays, blockArrays fills them
MR_JNI(jlongArray, blockMeta)(JNIEnv* env, jclass, jlong m, jint rid, jint cid) {
  mr_block_desc d{};
  if (throw_if(env, mr_matrix_get_block(ptr<mr_matrix>(m), rid, cid, &d))) return nullptr;
  return meta_of(env, d);
}
MR_JNI(void, blockArrays)(JNIEnv* env, jclass, jlong m, jint rid, jint cid, jintArray colPtrs, jintArray rowIndices, jdoubleArray values) {
  arrays_into(env, [&](mr_block_desc* d) { return mr_matrix_get_block(ptr<mr_matrix>(m), rid, cid, d); }, colPtrs, rowIndices, values);
}

// ---- operators, argument for argument with Dataset.scala:38-152
#define MR_JNI_BINARY(JNAME, CNAME)                                                                                       \
  MR_JNI(jlong, JNAME)(JNIEnv * env, jclass, jlong left, jlong leftRowNum, jlong leftColNum, jlong right, jlong rightRowNum, \
                       jlong rightColNum, jint blkSize) {                                                                 \
    mr_matrix* out = nullptr;                                                                                             \
    if (throw_if(env, CNAME(ptr<mr_matrix>(left), leftRowNum, leftColNum, ptr<mr_matrix>(right), rightRowNum, rightColNum, \
                            blkSize, &out)))                                                                              \
      return 0;                                                                                                           \
    return reinterpret_cast<jlong>(out);                                                                                  \
  }
MR_JNI_BINARY(matrixMultiply, mr_matrix_multiply)
MR_JNI_BINARY(addElement, mr_add_element)
MR_JNI_BINARY(multiplyElement, mr_multiply_element)
MR_JNI_BINARY(divideElement, mr_divide_element)
MR_JNI_BINARY(matrixRankOneUpdate, mr_rank_one_update)
MR_JNI(jlong, transpose)(JNIEnv* env, jclass, jlong a) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_transpose(ptr<mr_matrix>(a), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
#define MR_JNI_SCALAR(JNAME, CNAME)                                         \
  MR_JNI(jlong, JNAME)(JNIEnv * env, jclass, jlong a, jdouble alpha) {      \
    mr_matrix* out = nullptr;                                               \
    if (throw_if(env, CNAME(ptr<mr_matrix>(a), alpha, &out))) return 0;     \
    return reinterpret_cast<jlong>(out);                                    \
  }
MR_JNI_SCALAR(addScalar, mr_add_scalar)
MR_JNI_SCALAR(multiplyScalar, mr_multiply_scalar)
MR_JNI_SCALAR(power, mr_power)
// aggregates (Dataset.scala:63-82)
#define MR_JNI_AGG(JNAME, CNAME)                                                  \
  MR_JNI(jlong, JNAME)(JNIEnv * env, jclass, jlong a, jlong nrows, jlong ncols) { \
    mr_matrix* out = nullptr;                                                     \
    if (throw_if(env, CNAME(ptr<mr_matrix>(a), nrows, ncols, &out))) return 0;    \
    return reinterpret_cast<jlong>(out);                                          \
  }
MR_JNI_AGG(rowSum, mr_row_sum)
MR_JNI_AGG(colSum, mr_col_sum)
MR_JNI_AGG(sum, mr_sum)
MR_JNI_AGG(trace, mr_trace)
// slicing (Dataset.scala:38-55, 84-87)
MR_JNI(jlong, project)(JNIEnv* env, jclass, jlong a, jlong nrows, jlong ncols, jint blkSize, jboolean rowOrCol, jlong index) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_project(ptr<mr_matrix>(a), nrows, ncols, blkSize, rowOrCol ? 1 : 0, index, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, selection)(JNIEnv* env, jclass, jlong a, jlong nrows, jlong ncols, jint blkSize, jlong rowIdx, jlong colIdx) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_selection(ptr<mr_matrix>(a), nrows, ncols, blkSize, rowIdx, colIdx, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, vec)(JNIEnv* env, jclass, jlong a, jlong nrows, jlong ncols, jint blkSize) {
  mr_matrix* out = nullptr;
  if (throw_if(env, mr_vec(ptr<mr_matrix>(a), nrows, ncols, blkSize, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}

// ---- placement: Partitioner.getPartition of M/partitioner/*.scala, genBlockCyclicPartitioner (MatfastExecutionHelper.scala:46-62)
MR_JNI(jint, partitionId)(JNIEnv* env, jclass, jint scheme, jint p0, jint p1, jint p2, jint p3, jint rid, jint cid) {
  const int32_t params[4] = {p0, p1, p2, p3};
  int32_t out = -1;
  throw_if(env, mr_partition_id(scheme, params, rid, cid, &out));
  return out;
}
MR_JNI(jintArray, genBlockCyclic)(JNIEnv* env, jclass, jlong nrows, jlong ncols, jint blkSize) {
  int32_t p[4] = {0, 0, 0, 0};
  if (throw_if(env, mr_gen_block_cyclic(nrows, ncols, blkSize, p))) return nullptr;
  jintArray out = env->NewIntArray(4);
  if (out != nullptr) env->SetIntArrayRegion(out, 0, 4, p);
  return out;
}

// ---- one JVM driving all GPUs of the box (mr_init_grid): no executor JVMs, no MPI
MR_JNI(jlong, gridInit)(JNIEnv* env, jclass, jint ngpus, jboolean compat, jint gemmAlgo) {
  mr_options o{};
  o.device = -1;
  o.compat_bugs = compat ? 1 : 0;
  o.gemm_algo = gemmAlgo;
  mr_grid* g = nullptr;
  if (throw_if(env, mr_init_grid(&o, ngpus, &g))) return 0;
  return reinterpret_cast<jlong>(g);
}
MR_JNI(void, gridShutdown)(JNIEnv* env, jclass, jlong g) { throw_if(env, mr_grid_shutdown(ptr<mr_grid>(g))); }
MR_JNI(jlong, dmatrixCreate)(JNIEnv* env, jclass, jlong g, jlong nrows, jlong ncols, jint blkSize) {
  mr_dmatrix* m = nullptr;
  if (throw_if(env, mr_dmatrix_create(ptr<mr_grid>(g), nrows, ncols, blkSize, &m))) return 0;
  return reinterpret_cast<jlong>(m);
}
MR_JNI(void, dmatrixFree)(JNIEnv* env, jclass, jlong m) { throw_if(env, mr_dmatrix_free(ptr<mr_dmatrix>(m))); }
MR_JNI(void, dmatrixPutBlock)(JNIEnv* env, jclass, jlong m, jint rid, jint cid, jbyte type, jint numRows, jint numCols, jintArray colPtrs,
                              jintArray rowIndices, jdoubleArray values, jboolean isTransposed) {
  StagedBlock b(env, type, numRows, numCols, colPtrs, rowIndices, values, isTransposed);
  if (!b.ok) return;
  throw_if(env, mr_dmatrix_put_block(ptr<mr_dmatrix>(m), rid, cid, &b.d));  // routed to the GPU that owns (rid, cid)
}
MR_JNI(jboolean, dmatrixHasBlock)(JNIEnv* env, jclass, jlong m, jint rid, jint cid) {
  int32_t has = 0;
  throw_if(env, mr_dmatrix_has_block(ptr<mr_dmatrix>(m), rid, cid, &has));
  return has != 0;
}
MR_JNI(jlongArray, dmatrixBlockMeta)(JNIEnv* env, jclass, jlong m, jint rid, jint cid) {
  mr_block_desc d{};
  if (throw_if(env, mr_dmatrix_get_block(ptr<mr_dmatrix>(m), rid, cid, &d))) return nullptr;
  return meta_of(env, d);
}
MR_JNI(void, dmatrixBlockArrays)(JNIEnv* env, jclass, jlong m, jint rid, jint cid, jintArray colPtrs, jintArray rowIndices,
                                 jdoubleArray values) {
  arrays_into(env, [&](mr_block_desc* d) { return mr_dmatrix_get_block(ptr<mr_dmatrix>(m), rid, cid, d); }, colPtrs, rowIndices, values);
}
MR_JNI(jint, dmatrixOwner)(JNIEnv* env, jclass, jlong m, jint rid, jint cid) {
  int32_t rank = -1;
  throw_if(env, mr_dmatrix_owner(ptr<mr_dmatrix>(m), rid, cid, &rank));
  return rank;
}
MR_JNI(jlong, dmatrixMultiply)(JNIEnv* env, jclass, jlong a, jlong b) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_multiply(ptr<mr_dmatrix>(a), ptr<mr_dmatrix>(b), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixMultiplySplitK)(JNIEnv* env, jclass, jlong a, jlong b) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_multiply_ksplit(ptr<mr_dmatrix>(a), ptr<mr_dmatrix>(b), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixElementwise)(JNIEnv* env, jclass, jint op, jlong a, jlong b) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_elementwise(op, ptr<mr_dmatrix>(a), ptr<mr_dmatrix>(b), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jdouble, dmatrixReduceScalar)(JNIEnv* env, jclass, jlong a, jint what) {
  double v = 0.0;
  throw_if(env, mr_dmatrix_reduce_scalar(ptr<mr_dmatrix>(a), what, &v));
  return v;
}
MR_JNI(jlong, dmatrixRepartition)(JNIEnv* env, jclass, jlong a, jint newPr, jint newPc) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_repartition(ptr<mr_dmatrix>(a), newPr, newPc, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixTranspose)(JNIEnv* env, jclass, jlong a) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_transpose(ptr<mr_dmatrix>(a), &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixAxisSum)(JNIEnv* env, jclass, jlong a, jint axis) {  // 0 rowSum, 1 colSum
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_axis_sum(ptr<mr_dmatrix>(a), axis, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixProject)(JNIEnv* env, jclass, jlong a, jboolean rowOrCol, jlong index) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_project(ptr<mr_dmatrix>(a), rowOrCol ? 1 : 0, index, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixSelection)(JNIEnv* env, jclass, jlong a, jlong rowIdx, jlong colIdx) {
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_selection(ptr<mr_dmatrix>(a), rowIdx, colIdx, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}
MR_JNI(jlong, dmatrixScalar)(JNIEnv* env, jclass, jint op, jlong a, jdouble alpha) {  // 0 addScalar, 1 multiplyScalar, 2 power
  mr_dmatrix* out = nullptr;
  if (throw_if(env, mr_dmatrix_scalar(op, ptr<mr_dmatrix>(a), alpha, &out))) return 0;
  return reinterpret_cast<jlong>(out);
}

}  // extern "C"
#endif  // __has_include(<jni.h>)
