/*
 * marlin_b200_jni.c — the JNI veneer between edu.nju.pasalab.marlin.matrix.Native (scala/.../Native.scala) and the C ABI
 * of libmarlin_b200.so (include/marlin_b200.h).  One mechanical stub per @native: unwrap handles (jlong <-> pointer),
 * pin JVM arrays for the duration of the call (GetPrimitiveArrayCritical; nothing is retained), forward, and turn a
 * non-zero status into the exception the reference's Scala code throws in the same situation (`require` ->
 * IllegalArgumentException for bad arguments / dimension mismatch / unsupported grids, RuntimeException otherwise:
 * matrix/BlockMatrix.scala:90-91,132-133,150-151,189,192,218).
 *
 * Build (needs a JDK):  gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../include \
 *                           marlin_b200_jni.c -L../marlin_b200/lib -lmarlin_b200 -o libmarlin_b200_jni.so
 * This image has no JDK: without <jni.h> the file is compiled against jni_compile_check.h (types only, for gcc's
 * parser and type checker — tests/test_jni_veneer.py); such an object is never loaded anywhere.
 */
#if defined(__has_include)
#  if __has_include(<jni.h>)
#    include <jni.h>
#    define MB_HAVE_JNI 1
#  endif
#endif
#ifndef MB_HAVE_JNI
#  include "jni_compile_check.h"
#endif
#include <stdlib.h>
#include <string.h>
#include "marlin_b200.h"

#define NATIVE(ret, name) JNIEXPORT ret JNICALL Java_edu_nju_pasalab_marlin_matrix_Native_00024_##name
#define CTX(h) ((mb_ctx*)(intptr_t)(h))
#define BLK(h) ((mb_block*)(intptr_t)(h))
#define COMM(h) ((mb_comm*)(intptr_t)(h))

/* status -> exception (SURVEY 8b error convention) */
static void raise(JNIEnv* env, int32_t rc) {
    if (rc == MB_OK || (*env)->ExceptionCheck(env)) return;
    const char* cls = (rc == MB_ERR_INVALID_ARG || rc == MB_ERR_DIM_MISMATCH || rc == MB_ERR_UNSUPPORTED)
                          ? "java/lang/IllegalArgumentException"
                          : "java/lang/RuntimeException";
    (*env)->ThrowNew(env, (*env)->FindClass(env, cls), mb_last_error());
}

/* jlong[] of block handles -> malloc'd mb_block*[] (NULL entries stay NULL) */
static mb_block** handles(JNIEnv* env, jlongArray arr, jsize* n_out) {
    const jsize n = (*env)->GetArrayLength(env, arr);
    jlong* tmp = (jlong*)malloc(sizeof(jlong) * (size_t)(n > 0 ? n : 1));
    mb_block** out = (mb_block**)malloc(sizeof(mb_block*) * (size_t)(n > 0 ? n : 1));
    (*env)->GetLongArrayRegion(env, arr, 0, n, tmp);
    for (jsize i = 0; i < n; ++i) out[i] = BLK(tmp[i]);
    free(tmp);
    if (n_out) *n_out = n;
    return out;
}
static int32_t* ints(JNIEnv* env, jintArray arr) {
    const jsize n = (*env)->GetArrayLength(env, arr);
    int32_t* out = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    (*env)->GetIntArrayRegion(env, arr, 0, n, (jint*)out);
    return out;
}

/* ---- lifetime ---- */
NATIVE(jlong, init)(JNIEnv* e, jobject o, jint device) {
    mb_ctx* ctx = NULL;
    raise(e, mb_init(device, &ctx));
    return (jlong)(intptr_t)ctx;
}
NATIVE(void, shutdown)(JNIEnv* e, jobject o, jlong ctx) { raise(e, mb_shutdown(CTX(ctx))); }
NATIVE(void, synchronize)(JNIEnv* e, jobject o, jlong ctx) { raise(e, mb_synchronize(CTX(ctx))); }
NATIVE(jstring, version)(JNIEnv* e, jobject o) { return (*e)->NewStringUTF(e, mb_version()); }

/* ---- blocks: new SubMatrix(denseMatrix) / toBreeze (matrix/SubMatrix.scala:16-20, matrix/BlockMatrix.scala:70-85) ---- */
NATIVE(jlong, upload)(JNIEnv* e, jobject o, jlong ctx, jdoubleArray data, jint offset, jint rows, jint cols, jint majorStride,
                      jboolean isTranspose, jint storeAs) {
    mb_block* blk = NULL;
    jdouble* p = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, data, NULL);      /* JVM-owned, never retained */
    const int32_t rc = mb_block_upload(CTX(ctx), p, offset, rows, cols, majorStride, isTranspose ? 1 : 0, (mb_dtype)storeAs, &blk);
    (*e)->ReleasePrimitiveArrayCritical(e, data, p, JNI_ABORT);
    raise(e, rc);
    return (jlong)(intptr_t)blk;
}
NATIVE(void, download)(JNIEnv* e, jobject o, jlong ctx, jlong blk, jdoubleArray out, jint ld) {
    jdouble* p = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, out, NULL);
    const int32_t rc = mb_block_download(CTX(ctx), BLK(blk), p, ld);
    (*e)->ReleasePrimitiveArrayCritical(e, out, p, 0);
    raise(e, rc);
}
NATIVE(jlong, alloc)(JNIEnv* e, jobject o, jlong ctx, jint rows, jint cols, jint dtype) {
    mb_block* blk = NULL;
    raise(e, mb_block_alloc(CTX(ctx), rows, cols, (mb_dtype)dtype, &blk));
    return (jlong)(intptr_t)blk;
}
NATIVE(void, free)(JNIEnv* e, jobject o, jlong ctx, jlong blk) { raise(e, mb_block_free(CTX(ctx), BLK(blk))); }
NATIVE(jlong, viewT)(JNIEnv* e, jobject o, jlong ctx, jlong blk) {
    mb_block* out = NULL;
    raise(e, mb_block_view_t(CTX(ctx), BLK(blk), &out));
    return (jlong)(intptr_t)out;
}
NATIVE(jlong, slice)(JNIEnv* e, jobject o, jlong ctx, jlong blk, jint r0, jint r1, jint c0, jint c1) {
    mb_block* out = NULL;
    raise(e, mb_block_slice(CTX(ctx), BLK(blk), r0, r1, c0, c1, &out));
    return (jlong)(intptr_t)out;
}

/* ---- a1/a2/a9/a10: the per-block kernels (matrix/SubMatrix.scala:41-139, matrix/BlockMatrix.scala:514-523) ---- */
NATIVE(void, gemm)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong b, jlong c, jboolean accumulate) {
    raise(e, mb_block_gemm(CTX(ctx), BLK(a), BLK(b), BLK(c), accumulate ? 1 : 0));
}
NATIVE(void, add)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong b, jlong out) { raise(e, mb_block_add(CTX(ctx), BLK(a), BLK(b), BLK(out))); }
NATIVE(void, sub)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong b, jlong out) { raise(e, mb_block_sub(CTX(ctx), BLK(a), BLK(b), BLK(out))); }
NATIVE(void, hadamard)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong b, jlong out) {
    raise(e, mb_block_hadamard(CTX(ctx), BLK(a), BLK(b), BLK(out)));
}
NATIVE(void, axpb)(JNIEnv* e, jobject o, jlong ctx, jlong a, jdouble alpha, jdouble beta, jlong out) {
    raise(e, mb_block_axpb(CTX(ctx), BLK(a), alpha, beta, BLK(out)));
}
NATIVE(void, div)(JNIEnv* e, jobject o, jlong ctx, jlong a, jdouble b, jboolean bOverA, jlong out) {
    raise(e, mb_block_div(CTX(ctx), BLK(a), b, bOverA ? 1 : 0, BLK(out)));
}
NATIVE(void, transpose)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong out) { raise(e, mb_block_transpose(CTX(ctx), BLK(a), BLK(out))); }
NATIVE(void, copy)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong out) { raise(e, mb_block_copy(CTX(ctx), BLK(a), BLK(out))); }
NATIVE(jdouble, sum)(JNIEnv* e, jobject o, jlong ctx, jlong a) {
    double s = 0.0;
    raise(e, mb_block_sum(CTX(ctx), BLK(a), &s));
    return s;
}
NATIVE(void, gemv)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong x, jlong y, jboolean accumulate) {
    raise(e, mb_block_gemv(CTX(ctx), BLK(a), BLK(x), BLK(y), accumulate ? 1 : 0));
}
NATIVE(jdouble, dot)(JNIEnv* e, jobject o, jlong ctx, jlong x, jlong y) {
    double d = 0.0;
    raise(e, mb_block_dot(CTX(ctx), BLK(x), BLK(y), &d));
    return d;
}
NATIVE(void, ger)(JNIEnv* e, jobject o, jlong ctx, jlong x, jlong y, jlong out) { raise(e, mb_block_ger(CTX(ctx), BLK(x), BLK(y), BLK(out))); }
NATIVE(void, fillUniform)(JNIEnv* e, jobject o, jlong ctx, jlong blk, jlong partitionSeed, jlong first, jdouble lo, jdouble hi,
                          jboolean rowMajor) {
    raise(e, mb_fill_uniform(CTX(ctx), BLK(blk), partitionSeed, first, lo, hi, rowMajor ? 1 : 0));
}
/* ---- f4: the Breeze/LAPACK leaves of luDecompose / choleskyDecompose / inverse (matrix/DenseVecMatrix.scala:283-764) ---- */
NATIVE(void, lu)(JNIEnv* e, jobject o, jlong ctx, jlong a, jintArray permOut) {
    /* in place, dgetrf packing; permOut (rows entries) = the reference's permutation array: row i of L*U is row perm[i] of A */
    const jsize n = (*e)->GetArrayLength(e, permOut);
    int32_t* perm = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    const int32_t rc = mb_block_lu(CTX(ctx), BLK(a), perm);
    if (rc == MB_OK) (*e)->SetIntArrayRegion(e, permOut, 0, n, (const jint*)perm);
    free(perm);
    raise(e, rc);
}
NATIVE(void, cholesky)(JNIEnv* e, jobject o, jlong ctx, jlong a) { raise(e, mb_block_cholesky(CTX(ctx), BLK(a))); }
NATIVE(void, inverse)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong out) { raise(e, mb_block_inverse(CTX(ctx), BLK(a), BLK(out))); }
/* ---- f5: the local steps of computeSVD (matrix/DenseVecMatrix.scala:1464-1486, 1565-1621) ---- */
NATIVE(void, gramian)(JNIEnv* e, jobject o, jlong ctx, jlong a, jlong g) { raise(e, mb_block_gramian(CTX(ctx), BLK(a), BLK(g))); }
NATIVE(jint, syev)(JNIEnv* e, jobject o, jlong ctx, jlong g, jlong v, jdoubleArray wOut) {
    /* wOut (n entries): eigenvalues by |w| descending; returns the number of Jacobi sweeps */
    const jsize n = (*e)->GetArrayLength(e, wOut);
    double* w = (double*)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
    int32_t sweeps = 0;
    const int32_t rc = mb_block_syev(CTX(ctx), BLK(g), BLK(v), w, &sweeps);
    if (rc == MB_OK && n > 0) {
        double* dst = (double*)(*e)->GetPrimitiveArrayCritical(e, wOut, NULL);
        memcpy(dst, w, sizeof(double) * (size_t)n);
        (*e)->ReleasePrimitiveArrayCritical(e, wOut, dst, 0);
    }
    free(w);
    raise(e, rc);
    return sweeps;
}
NATIVE(jint, svdMode)(JNIEnv* e, jobject o, jlong n, jint k, jstring mode) {
    const char* m = (*e)->GetStringUTFChars(e, mode, NULL);
    int32_t cm = 0;
    const int32_t rc = mb_svd_mode(n, k, m, &cm);
    (*e)->ReleaseStringUTFChars(e, mode, m);
    raise(e, rc);
    return cm;
}
NATIVE(jint, svdRank)(JNIEnv* e, jobject o, jdoubleArray sigmas, jint k, jdouble rCond) {
    const jsize n = (*e)->GetArrayLength(e, sigmas);
    double* s = (double*)(*e)->GetPrimitiveArrayCritical(e, sigmas, NULL);
    const int32_t sk = mb_svd_rank(s, n, k, rCond);
    (*e)->ReleasePrimitiveArrayCritical(e, sigmas, s, JNI_ABORT);
    if (sk < 0) raise(e, sk);
    return sk;
}
NATIVE(void, trsm)(JNIEnv* e, jobject o, jlong ctx, jlong t, jboolean lower, jboolean unitDiagonal, jlong b) {
    raise(e, mb_block_trsm(CTX(ctx), BLK(t), lower ? 1 : 0, unitDiagonal ? 1 : 0, BLK(b)));
}
NATIVE(void, setFp64Mode)(JNIEnv* e, jobject o, jlong ctx, jint mode, jint slices) { raise(e, mb_set_fp64_mode(CTX(ctx), mode, slices)); }

/* ---- a3-a6: whole multiplies on one GPU ---- */
NATIVE(void, matmulBlocked)(JNIEnv* e, jobject o, jlong ctx, jlongArray aTiles, jlongArray bTiles, jint m, jint k, jint n,
                            jlongArray cTiles) {
    mb_block **a = handles(e, aTiles, NULL), **b = handles(e, bTiles, NULL), **c = handles(e, cTiles, NULL);
    raise(e, mb_matmul_blocked(CTX(ctx), a, b, m, k, n, c));
    free(a); free(b); free(c);
}
NATIVE(void, matmulRowsharded)(JNIEnv* e, jobject o, jlong ctx, jlong aRows, jlong b, jlong cRows) {
    raise(e, mb_matmul_rowsharded(CTX(ctx), BLK(aRows), BLK(b), BLK(cRows)));
}
NATIVE(void, matmulRowshardedHost)(JNIEnv* e, jobject o, jlong ctx, jdoubleArray aRows, jlong rows, jint k, jdoubleArray b, jint n,
                                   jdoubleArray cRows) {
    /* the partition's packed rowsMat (matrix/DenseVecMatrix.scala:1672-1675), the broadcast matrix, the result rows */
    jdouble* pa = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, aRows, NULL);
    jdouble* pb = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, b, NULL);
    jdouble* pc = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, cRows, NULL);
    const int32_t rc = mb_matmul_rowsharded_host(CTX(ctx), pa, rows, k, pb, n, pc);
    (*e)->ReleasePrimitiveArrayCritical(e, cRows, pc, 0);
    (*e)->ReleasePrimitiveArrayCritical(e, b, pb, JNI_ABORT);
    (*e)->ReleasePrimitiveArrayCritical(e, aRows, pa, JNI_ABORT);
    raise(e, rc);
}
/* the netlib seam: com.github.fommil.netlib.BLAS.dgemm with JVM arrays (INTEGRATION.md section 2) */
NATIVE(void, dgemmHost)(JNIEnv* e, jobject o, jlong ctx, jboolean transA, jboolean transB, jint m, jint n, jint k, jdouble alpha,
                        jdoubleArray a, jint aOff, jint lda, jdoubleArray b, jint bOff, jint ldb, jdouble beta, jdoubleArray c,
                        jint cOff, jint ldc) {
    jdouble* pa = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, a, NULL);
    jdouble* pb = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, b, NULL);
    jdouble* pc = (jdouble*)(*e)->GetPrimitiveArrayCritical(e, c, NULL);
    const int32_t rc = mb_dgemm_host(CTX(ctx), transA ? 'T' : 'N', transB ? 'T' : 'N', m, n, k, alpha, pa, aOff, lda, pb, bOff, ldb,
                                     beta, pc, cOff, ldc);
    (*e)->ReleasePrimitiveArrayCritical(e, c, pc, 0);
    (*e)->ReleasePrimitiveArrayCritical(e, b, pb, JNI_ABORT);
    (*e)->ReleasePrimitiveArrayCritical(e, a, pa, JNI_ABORT);
    raise(e, rc);
}

/* ---- (e): BlockMatrix.multiply across the GPUs of one box (matrix/BlockMatrix.scala:159-178) ---- */
NATIVE(jlong, commInit)(JNIEnv* e, jobject o, jlong ctx, jint rank, jint world, jstring session) {
    mb_comm* comm = NULL;
    const char* s = (*e)->GetStringUTFChars(e, session, NULL);
    const int32_t rc = mb_comm_init(CTX(ctx), rank, world, s, &comm);
    (*e)->ReleaseStringUTFChars(e, session, s);
    raise(e, rc);
    return (jlong)(intptr_t)comm;
}
NATIVE(void, commDestroy)(JNIEnv* e, jobject o, jlong comm) { raise(e, mb_comm_destroy(COMM(comm))); }
NATIVE(void, commBarrier)(JNIEnv* e, jobject o, jlong comm) { raise(e, mb_comm_barrier(COMM(comm))); }
NATIVE(void, commCheck)(JNIEnv* e, jobject o, jlong comm) { raise(e, mb_comm_check(COMM(comm))); }
NATIVE(void, commAbort)(JNIEnv* e, jobject o, jlong comm) { raise(e, mb_comm_abort(COMM(comm))); }
NATIVE(jintArray, distPlan)(JNIEnv* e, jobject o, jint m, jint k, jint n, jint world) {
    /* returns m*k*n product ranks followed by m*n C-tile owners */
    const jsize np = m * k * n, nc = m * n;
    int32_t* buf = (int32_t*)malloc(sizeof(int32_t) * (size_t)(np + nc > 0 ? np + nc : 1));
    const int32_t rc = mb_dist_plan(m, k, n, world, buf, buf + np);
    jintArray out = NULL;
    if (rc == MB_OK) {
        out = (*e)->NewIntArray(e, np + nc);
        (*e)->SetIntArrayRegion(e, out, 0, np + nc, (const jint*)buf);
    }
    free(buf);
    raise(e, rc);
    return out;
}
NATIVE(void, matmulBlockedDist)(JNIEnv* e, jobject o, jlong comm, jlongArray aTiles, jintArray aOwner, jlongArray bTiles,
                                jintArray bOwner, jint m, jint k, jint n, jintArray rowLen, jintArray kLen, jintArray colLen,
                                jint dtype, jlongArray cTiles) {
    mb_block **a = handles(e, aTiles, NULL), **b = handles(e, bTiles, NULL), **c = handles(e, cTiles, NULL);
    int32_t *ao = ints(e, aOwner), *bo = ints(e, bOwner), *rl = ints(e, rowLen), *kl = ints(e, kLen), *cl = ints(e, colLen);
    raise(e, mb_matmul_blocked_dist(COMM(comm), a, ao, b, bo, m, k, n, rl, kl, cl, dtype, c));
    free(a); free(b); free(c); free(ao); free(bo); free(rl); free(kl); free(cl);
}

/* ---- a7/a8/a11: driver-side integer logic (utils/MTUtils.scala:18-21,150-213; rdd/MatrixMultPartitioner.scala, rdd/MatrixElemOpPartitioner.scala) ---- */
NATIVE(jintArray, chooseSplit)(JNIEnv* e, jobject o, jlong m, jlong k, jlong n, jint cores) {
    int32_t mkn[3] = {0, 0, 0};
    raise(e, mb_choose_split(m, k, n, cores, mkn));
    jintArray out = (*e)->NewIntArray(e, 3);
    (*e)->SetIntArrayRegion(e, out, 0, 3, (const jint*)mkn);
    return out;
}
NATIVE(jintArray, chooseStrategy)(JNIEnv* e, jobject o, jlong aRows, jlong aCols, jlong bCols, jint cores, jint thresholdMb,
                                  jboolean otherIsBlock) {
    int32_t res[4] = {0, 0, 0, 0};                       /* strategy, m, k, n */
    raise(e, mb_choose_strategy(aRows, aCols, bCols, cores, thresholdMb, otherIsBlock ? 1 : 0, &res[0], &res[1]));
    jintArray out = (*e)->NewIntArray(e, 4);
    (*e)->SetIntArrayRegion(e, out, 0, 4, (const jint*)res);
    return out;
}
NATIVE(jint, multPartition)(JNIEnv* e, jobject o, jint i, jint j, jint kk, jint m, jint k, jint n) {
    return mb_mult_partition(i, j, kk, m, k, n);
}
NATIVE(jint, elemPartition)(JNIEnv* e, jobject o, jint row, jint col, jint blksByCol) { return mb_elem_partition(row, col, blksByCol); }
NATIVE(jintArray, blockLen)(JNIEnv* e, jobject o, jlong total, jint parts) {
    int32_t res[2] = {0, 0};
    raise(e, mb_block_len(total, parts, &res[0], &res[1]));
    jintArray out = (*e)->NewIntArray(e, 2);
    (*e)->SetIntArrayRegion(e, out, 0, 2, (const jint*)res);
    return out;
}
NATIVE(jlong, hashSeed)(JNIEnv* e, jobject o, jlong seed) { return mb_hash_seed(seed); }
NATIVE(jlongArray, partitionSeeds)(JNIEnv* e, jobject o, jlong seed, jint numPartitions) {
    int64_t* buf = (int64_t*)malloc(sizeof(int64_t) * (size_t)(numPartitions > 0 ? numPartitions : 1));
    const int32_t rc = mb_partition_seeds(seed, numPartitions, buf);
    jlongArray out = NULL;
    if (rc == MB_OK) {
        out = (*e)->NewLongArray(e, numPartitions);
        (*e)->SetLongArrayRegion(e, out, 0, numPartitions, (const jlong*)buf);
    }
    free(buf);
    raise(e, rc);
    return out;
}
