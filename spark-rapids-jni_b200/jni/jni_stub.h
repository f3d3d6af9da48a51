/* jni_stub.h -- the handful of <jni.h> declarations the shim uses, for syntax-checking it in an image without a JDK
 * (g++ -fsyntax-only -DSRJ_JNI_STUBS).  A real build includes the JDK's <jni.h> instead. */
#pragma once
#include <cstdint>
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
typedef int32_t jint;
typedef int64_t jlong;
typedef double jdouble;
typedef uint8_t jboolean;
typedef int32_t jsize;
class _jobject {};
typedef _jobject* jobject;
typedef jobject jclass;
typedef jobject jthrowable;
typedef jobject jarray;
typedef jarray jintArray;
typedef jarray jlongArray;
typedef jarray jdoubleArray;
typedef jobject jstring;
struct JNIEnv {
  const char* GetStringUTFChars(jstring, jboolean*);
  void ReleaseStringUTFChars(jstring, const char*);
  jclass FindClass(const char*);
  jint ThrowNew(jclass, const char*);
  jint Throw(jthrowable);
  jboolean ExceptionCheck();
  jsize GetArrayLength(jarray);
  jint* GetIntArrayElements(jintArray, jboolean*);
  void ReleaseIntArrayElements(jintArray, jint*, jint);
  jlong* GetLongArrayElements(jlongArray, jboolean*);
  void ReleaseLongArrayElements(jlongArray, jlong*, jint);
  jdouble* GetDoubleArrayElements(jdoubleArray, jboolean*);
  void ReleaseDoubleArrayElements(jdoubleArray, jdouble*, jint);
  jlongArray NewLongArray(jsize);
  void SetLongArrayRegion(jlongArray, jsize, jsize, const jlong*);
  jintArray NewIntArray(jsize);
  void SetIntArrayRegion(jintArray, jsize, jsize, const jint*);
  struct _jmethodID* GetMethodID(jclass, const char*, const char*);
  jobject NewObject(jclass, struct _jmethodID*, ...);
  jstring NewStringUTF(const char*);
};
typedef struct _jmethodID* jmethodID;
#define JNI_ABORT 2
