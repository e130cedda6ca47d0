/* jni/stub/jni.h — a minimal stand-in for the JDK's <jni.h>, ONLY for `g++ -fsyntax-only` checks of
 * jni/paimon_gpu_jni.cc in images without a JDK (this one has none).  It declares the JNI types and the JNIEnv
 * member functions the shim uses, with the signatures of the JNI specification; it is never linked or shipped.
 * Build the real shim against $JAVA_HOME/include/jni.h. */
#ifndef PAIMON_GPU_JNI_STUB_H
#define PAIMON_GPU_JNI_STUB_H
#include <stdint.h>
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
#define JNI_ABORT 2
typedef int32_t jint;
typedef int64_t jlong;
typedef int8_t jbyte;
typedef uint8_t jboolean;
typedef float jfloat;
typedef double jdouble;
typedef jint jsize;
class _jobject {};
typedef _jobject *jobject;
typedef jobject jclass;
typedef jobject jstring;
typedef jobject jarray;
typedef jobject jobjectArray;
typedef jobject jintArray;
typedef jobject jlongArray;
typedef jobject jbooleanArray;
typedef jobject jdoubleArray;
typedef jobject jthrowable;
struct JNIEnv {
    jclass FindClass(const char *name);
    jint ThrowNew(jclass clazz, const char *msg);
    jsize GetArrayLength(jarray array);
    jobject GetObjectArrayElement(jobjectArray array, jsize index);
    void GetIntArrayRegion(jintArray array, jsize start, jsize len, jint *buf);
    void SetIntArrayRegion(jintArray array, jsize start, jsize len, const jint *buf);
    void GetLongArrayRegion(jlongArray array, jsize start, jsize len, jlong *buf);
    void SetLongArrayRegion(jlongArray array, jsize start, jsize len, const jlong *buf);
    void GetBooleanArrayRegion(jbooleanArray array, jsize start, jsize len, jboolean *buf);
    jlongArray NewLongArray(jsize len);
    jintArray NewIntArray(jsize len);
    jdoubleArray NewDoubleArray(jsize len);
    void SetDoubleArrayRegion(jdoubleArray array, jsize start, jsize len, const jdouble *buf);
    void GetDoubleArrayRegion(jdoubleArray array, jsize start, jsize len, jdouble *buf);
    void *GetDirectBufferAddress(jobject buf);
    jlong GetDirectBufferCapacity(jobject buf);
    const char *GetStringUTFChars(jstring str, jboolean *isCopy);
    void ReleaseStringUTFChars(jstring str, const char *chars);
    jstring NewStringUTF(const char *utf);
};
#endif
