/* NOT the JNI.  A just-enough declaration of the JNI types and the JNIEnv entries marlin_b200_jni.c uses, so that the
 * veneer is at least parsed and type-checked by gcc in images without a JDK (tests/test_jni_veneer.py).  The function
 * table below does not have the real layout: objects built against this header must never be loaded into a JVM.  With
 * a JDK present, marlin_b200_jni.c includes the real <jni.h> and this file is not used. */
#ifndef MARLIN_B200_JNI_COMPILE_CHECK_H
#define MARLIN_B200_JNI_COMPILE_CHECK_H
#include <stdint.h>
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
#define JNI_ABORT 2
#define JNI_FALSE 0
#define JNI_TRUE 1
typedef int32_t jint;
typedef int64_t jlong;
typedef double jdouble;
typedef float jfloat;
typedef uint8_t jboolean;
typedef jint jsize;
typedef void* jobject;
typedef jobject jclass;
typedef jobject jstring;
typedef jobject jarray;
typedef jarray jdoubleArray;
typedef jarray jintArray;
typedef jarray jlongArray;
typedef jarray jfloatArray;
struct JNINativeInterface_;
typedef const struct JNINativeInterface_* JNIEnv;
struct JNINativeInterface_ {
    jclass (*FindClass)(JNIEnv*, const char*);
    jint (*ThrowNew)(JNIEnv*, jclass, const char*);
    jboolean (*ExceptionCheck)(JNIEnv*);
    void* (*GetPrimitiveArrayCritical)(JNIEnv*, jarray, jboolean*);
    void (*ReleasePrimitiveArrayCritical)(JNIEnv*, jarray, void*, jint);
    jsize (*GetArrayLength)(JNIEnv*, jarray);
    jintArray (*NewIntArray)(JNIEnv*, jsize);
    jlongArray (*NewLongArray)(JNIEnv*, jsize);
    void (*SetIntArrayRegion)(JNIEnv*, jintArray, jsize, jsize, const jint*);
    void (*SetLongArrayRegion)(JNIEnv*, jlongArray, jsize, jsize, const jlong*);
    void (*GetIntArrayRegion)(JNIEnv*, jintArray, jsize, jsize, jint*);
    void (*GetLongArrayRegion)(JNIEnv*, jlongArray, jsize, jsize, jlong*);
    void (*GetFloatArrayRegion)(JNIEnv*, jfloatArray, jsize, jsize, jfloat*);
    void (*GetDoubleArrayRegion)(JNIEnv*, jdoubleArray, jsize, jsize, jdouble*);
    void (*SetDoubleArrayRegion)(JNIEnv*, jdoubleArray, jsize, jsize, const jdouble*);
    const char* (*GetStringUTFChars)(JNIEnv*, jstring, jboolean*);
    void (*ReleaseStringUTFChars)(JNIEnv*, jstring, const char*);
    jstring (*NewStringUTF)(JNIEnv*, const char*);
};
#endif
