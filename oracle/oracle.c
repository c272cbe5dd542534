/*
 * oracle.c -- C restatement of the reference's dense block-multiply algorithm (TEST INFRASTRUCTURE:
 * only tests/ and bench.py's cpu_baseline leg may load this; PARITY UNPINNED, see matrel_oracle.py).
 *
 * Restates, for all-dense column-major blocks:
 *   matrixMultiplyGeneral   <reference>/src/main/scala/org/apache/spark/sql/matfast/execution/MatfastExecutionHelper.scala:235-263
 *   MLMatrix.multiply       .../matrix/MLMatrix.scala:100-104   (fresh zeroed C, gemm(1.0, A, B, 0.0, C))
 *   BLAS.gemmddd -> dgemm   .../matrix/BLAS.scala:327-346
 *   LocalMatrix.addDense    .../matrix/LocalMatrix.scala:56-63  (two toArray copies + a third array)
 *   MLMatrixSerializer      .../util/MLMatrixSerializer.scala:26-69 (copy in / copy out)
 * dgemm is the reference-BLAS loop nest (what netlib-java's pure-JVM F2jBLAS executes when no native
 * BLAS is installed, i.e. stock Spark 2.1.0): for j, for l, temp = B(l,j), for i: C(i,j) += temp*A(i,l).
 * One task per output block, OpenMP threads = Spark local[*] task slots.
 *
 * Build: gcc -O3 -march=x86-64-v3 -fopenmp -shared -fPIC oracle/oracle.c -o oracle/liboracle.so -lm
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* java.util.Random (48-bit LCG) */
typedef struct { uint64_t s; } jrand;
static void jr_seed(jrand* r, int64_t seed) { r->s = ((uint64_t)seed ^ 0x5DEECE66DULL) & ((1ULL << 48) - 1); }
static uint32_t jr_next(jrand* r, int bits) {
  r->s = (r->s * 0x5DEECE66DULL + 0xBULL) & ((1ULL << 48) - 1);
  return (uint32_t)(r->s >> (48 - bits));
}
static double jr_double(jrand* r) {
  uint64_t hi = jr_next(r, 26), lo = jr_next(r, 27);
  return (double)((hi << 27) + lo) * (1.0 / 9007199254740992.0);
}

/* DenseMatrix.rand(rows, cols, new Random(seed)) -- column-major fill in storage order */
void oracle_rand_block(double* out, int64_t n, int64_t seed) {
  jrand r;
  jr_seed(&r, seed);
  for (int64_t i = 0; i < n; ++i) out[i] = jr_double(&r);
}

/* reference BLAS dgemm, "N","N", alpha = 1, beta = 0 into a zeroed C (column-major) */
void oracle_dgemm_f2j(int m, int n, int k, const double* A, int lda, const double* B, int ldb, double* C, int ldc) {
  for (int j = 0; j < n; ++j) {
    for (int i = 0; i < m; ++i) C[i + (size_t)ldc * j] = 0.0;
    for (int l = 0; l < k; ++l) {
      const double temp = B[l + (size_t)ldb * j];
      if (temp != 0.0) {
        const double* a = A + (size_t)lda * l;
        double* c = C + (size_t)ldc * j;
        for (int i = 0; i < m; ++i) c[i] += temp * a[i];
      }
    }
  }
}

/*
 * C = A * B for nb x nb grids of blk x blk blocks (A[i*nb + k], B[k*nb + j], C[i*nb + j] are pointers to
 * column-major blocks), computing the first `ntasks` output blocks in row-major (i, j) order; nk > 0 limits
 * the k loop to the first nk block pairs (bounded timing samples).
 * Per pair: copy-in of both operands, fresh zeroed product, dgemm, add into the running sum with the
 * reference's allocation pattern; copy-out at the end.  Returns 0 on success.
 */
int oracle_block_multiply_f2j(int nb, int blk, const double* const* A, const double* const* B, double* const* C,
                              int ntasks, int threads, int nk) {
  const size_t bb = (size_t)blk * blk;
  int fail = 0;
#ifdef _OPENMP
  if (threads > 0) omp_set_num_threads(threads);
#endif
#pragma omp parallel for schedule(dynamic, 1)
  for (int t = 0; t < ntasks; ++t) {
    const int i = t / nb, j = t % nb;
    double* a = (double*)malloc(bb * sizeof(double));
    double* b = (double*)malloc(bb * sizeof(double));
    double* p = (double*)malloc(bb * sizeof(double));
    double* acc = (double*)malloc(bb * sizeof(double));
    double* sum = (double*)malloc(bb * sizeof(double));
    if (!a || !b || !p || !acc || !sum) {
      fail = 1;
    } else {
      for (int k = 0; k < (nk > 0 && nk < nb ? nk : nb); ++k) {
        memcpy(a, A[(size_t)i * nb + k], bb * sizeof(double)); /* deserialize */
        memcpy(b, B[(size_t)k * nb + j], bb * sizeof(double));
        oracle_dgemm_f2j(blk, blk, blk, a, blk, b, blk, p, blk);
        if (k == 0) {
          memcpy(acc, p, bb * sizeof(double));
        } else { /* addDense: arr(i) = arr1(i) + arr2(i) into a third array */
          for (size_t e = 0; e < bb; ++e) sum[e] = acc[e] + p[e];
          double* tmp = acc; acc = sum; sum = tmp;
        }
      }
      memcpy(C[(size_t)i * nb + j], acc, bb * sizeof(double)); /* serialize */
    }
    free(a); free(b); free(p); free(acc); free(sum);
  }
  return fail;
}

int oracle_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
