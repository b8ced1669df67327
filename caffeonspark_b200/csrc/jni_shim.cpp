// jni_shim.cpp -- the com.yahoo.ml.jcaffe.CaffeNet natives over the C ABI.
//
// Replaces caffe-distri/src/main/cpp/jni/JniCaffeNet.cpp (18 exports) one for
// one; helper conventions follow caffe-distri/src/main/cpp/common.cpp
// (native pointer in BaseObject.address via init(J)V :8-34 / GetFieldID
// "address" :36-55, null-tolerant string arrays :57-77, C++ failure ->
// java.lang.Exception :111-121).  Compiled only where a JDK provides <jni.h>
// (the build container has none, so this file is NOT part of the tested
// surface: tests bind the C ABI directly; see INTEGRATION.md).
//
// FloatBlob stays the reference's class: the shim reads the host pointer and
// element count through its public Java API (FloatBlob.cpu_data() ->
// FloatArray.arrayAddress, FloatBlob.count()) and passes plain pointers down.
#if defined(__has_include)
#if __has_include(<jni.h>)
#define COS_HAVE_JNI 1
#endif
#endif

#ifdef COS_HAVE_JNI
#include <jni.h>

#include <string>
#include <vector>

#include "../../include/caffedistri_b200.h"

namespace {

void throw_java(JNIEnv* env, const char* msg) {  // common.cpp:118-121 ThrowCosJavaException
  jclass ex = env->FindClass("java/lang/Exception");
  if (ex) env->ThrowNew(ex, msg);
}

cos_net* native(JNIEnv* env, jobject self) {  // common.cpp:36-55 GetNativeAddress
  if (!self) return nullptr;
  jclass c = env->GetObjectClass(self);
  jfieldID f = c ? env->GetFieldID(c, "address", "J") : nullptr;
  if (!f || env->ExceptionCheck()) return nullptr;
  return reinterpret_cast<cos_net*>(env->GetLongField(self, f));
}

bool set_native(JNIEnv* env, jobject self, void* p) {  // common.cpp:8-34 SetNativeAddress
  jclass c = env->GetObjectClass(self);
  jmethodID m = c ? env->GetMethodID(c, "init", "(J)V") : nullptr;
  if (!m || env->ExceptionCheck()) return false;
  env->CallVoidMethod(self, m, reinterpret_cast<jlong>(p));
  return !env->ExceptionCheck();
}

struct Utf {  // RAII GetStringUTFChars
  JNIEnv* env; jstring s; const char* c;
  Utf(JNIEnv* e, jstring js) : env(e), s(js), c(js ? e->GetStringUTFChars(js, nullptr) : nullptr) {}
  ~Utf() { if (c) env->ReleaseStringUTFChars(s, c); }
};

jobjectArray to_java_strings(JNIEnv* env, const char* const* v, int n) {
  jclass sc = env->FindClass("java/lang/String");
  jobjectArray arr = env->NewObjectArray(n, sc, nullptr);
  for (int i = 0; arr && i < n; ++i) {
    jstring s = env->NewStringUTF(v[i] ? v[i] : "");
    env->SetObjectArrayElement(arr, i, s);
    env->DeleteLocalRef(s);
  }
  return arr;
}

// FloatBlob[] -> cos_blob[] through the reference's Java API
bool blobs_from_java(JNIEnv* env, jobjectArray data, std::vector<cos_blob>* out) {
  const jsize n = env->GetArrayLength(data);
  out->resize(n);
  for (jsize i = 0; i < n; ++i) {
    jobject b = env->GetObjectArrayElement(data, i);
    if (!b) return false;
    jclass bc = env->GetObjectClass(b);
    jmethodID count = env->GetMethodID(bc, "count", "()I");
    jmethodID cpu = env->GetMethodID(bc, "cpu_data", "()Lcom/yahoo/ml/jcaffe/FloatArray;");
    if (!count || !cpu) return false;
    const jint cnt = env->CallIntMethod(b, count);
    jobject arr = env->CallObjectMethod(b, cpu);
    if (!arr || env->ExceptionCheck()) return false;
    jfieldID af = env->GetFieldID(env->GetObjectClass(arr), "arrayAddress", "J");
    if (!af) return false;
    (*out)[i].data = reinterpret_cast<const float*>(env->GetLongField(arr, af));
    (*out)[i].num = cnt;  // flat: the gradient producer knows the input shape from the net definition
    (*out)[i].channels = (*out)[i].height = (*out)[i].width = 1;
    env->DeleteLocalRef(arr);
    env->DeleteLocalRef(b);
  }
  return true;
}

}  // namespace

extern "C" {

// (Ljava/lang/String;Ljava/lang/String;Ljava/lang/String;IIIZIII)Z   JniCaffeNet.cpp:14-89
JNIEXPORT jboolean JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_allocate(
    JNIEnv* env, jobject self, jstring solver, jstring model, jstring state, jint num_local_devices,
    jint cluster_size, jint rank, jboolean is_training, jint connection_type, jint start_device_id,
    jint validation_net_id) {
  Utf s(env, solver), m(env, model), st(env, state);
  if (!s.c) return JNI_FALSE;
  cos_net* net = nullptr;
  if (!cos_net_allocate(s.c, m.c, st.c, num_local_devices, cluster_size, rank, is_training, connection_type,
                        start_device_id, validation_net_id, &net)) {
    throw_java(env, cos_last_error());
    return JNI_FALSE;
  }
  // train() needs a gradient producer: attach the built-in one when it can run this net (DESIGN.md section 14),
  // filling the weights from the prototxt unless a model file was restored.  A net it refuses behaves as before:
  // train() then fails until a producer is registered.
  if (is_training) cos_net_use_native_producer(net, nullptr, (m.c && *m.c) ? 0 : 1);
  return set_native(env, self, net) ? JNI_TRUE : JNI_FALSE;
}

// (J)V   JniCaffeNet.cpp:96-99
JNIEXPORT void JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_deallocate(JNIEnv*, jobject, jlong address) {
  cos_net_deallocate(reinterpret_cast<cos_net*>(address));
}

// ()[Ljava/lang/String;   JniCaffeNet.cpp:106-159
JNIEXPORT jobjectArray JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_localAddresses(JNIEnv* env, jobject self) {
  const char* const* v = nullptr;
  int n = cos_net_local_addresses(native(env, self), &v);
  if (n < 0) return nullptr;
  return to_java_strings(env, v, n);
}

// ()Z   JniCaffeNet.cpp:166-177
JNIEXPORT jboolean JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_sync(JNIEnv* env, jobject self) {
  if (cos_net_sync(native(env, self))) return JNI_TRUE;
  throw_java(env, cos_last_error());
  return JNI_FALSE;
}

// ([Ljava/lang/String;)Z   JniCaffeNet.cpp:184-228
JNIEXPORT jboolean JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_connect(JNIEnv* env, jobject self, jobjectArray addrs) {
  std::vector<std::string> store;
  std::vector<const char*> ptrs;
  const jsize n = addrs ? env->GetArrayLength(addrs) : 0;
  store.resize(n);
  for (jsize i = 0; i < n; ++i) {
    jstring js = static_cast<jstring>(env->GetObjectArrayElement(addrs, i));
    if (js) {
      Utf u(env, js);
      store[i] = u.c ? u.c : "";
      ptrs.push_back(store[i].c_str());
      env->DeleteLocalRef(js);
    } else {
      ptrs.push_back(nullptr);  // null entries are allowed (common.cpp:57-77)
    }
  }
  return cos_net_connect(native(env, self), n ? ptrs.data() : nullptr, n) ? JNI_TRUE : JNI_FALSE;
}

// (I)I   JniCaffeNet.cpp:235-249
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_deviceID(JNIEnv* env, jobject self, jint idx) {
  return cos_net_device_id(native(env, self), idx);
}

// (IZ)Z   JniCaffeNet.cpp:256-270
JNIEXPORT jboolean JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_init(JNIEnv* env, jobject self, jint idx,
                                                                 jboolean enable_nn) {
  return cos_net_init(native(env, self), idx, enable_nn) ? JNI_TRUE : JNI_FALSE;
}

// (I[Lcom/yahoo/ml/jcaffe/FloatBlob;[Ljava/lang/String;)[Lcom/yahoo/ml/jcaffe/FloatBlob;   JniCaffeNet.cpp:277-376
JNIEXPORT jobjectArray JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_predict(JNIEnv* env, jobject, jint, jobjectArray,
                                                                        jobjectArray) {
  cos_net_predict(nullptr, 0, nullptr, 0, nullptr, 0, nullptr);
  throw_java(env, cos_last_error());
  return nullptr;
}

// (I[Lcom/yahoo/ml/jcaffe/FloatBlob;)Z   JniCaffeNet.cpp:383-413
JNIEXPORT jboolean JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_train(JNIEnv* env, jobject self, jint idx,
                                                                  jobjectArray data) {
  if (!data) {
    throw_java(env, "data is NULL");
    return JNI_FALSE;
  }
  std::vector<cos_blob> blobs;
  if (!blobs_from_java(env, data, &blobs)) {
    throw_java(env, "could not read FloatBlob[]");
    return JNI_FALSE;
  }
  if (cos_net_train(native(env, self), idx, blobs.data(), static_cast<int>(blobs.size()))) return JNI_TRUE;
  throw_java(env, cos_last_error());
  return JNI_FALSE;
}

// ([Lcom/yahoo/ml/jcaffe/FloatBlob;)V and ()V   JniCaffeNet.cpp:420-470
JNIEXPORT void JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_validation(JNIEnv* env, jobject, jobjectArray) {
  cos_net_validation(nullptr, nullptr, 0);
  throw_java(env, cos_last_error());
}
JNIEXPORT void JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_aggregateValidationOutputs(JNIEnv* env, jobject) {
  cos_net_aggregate_validation_outputs(nullptr);
  throw_java(env, cos_last_error());
}

// (I)I x3, ()I x2   JniCaffeNet.cpp:479-580
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getInitIter(JNIEnv* env, jobject self, jint idx) {
  return cos_net_get_init_iter(native(env, self), idx);
}
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getMaxIter(JNIEnv* env, jobject self, jint idx) {
  return cos_net_get_max_iter(native(env, self), idx);
}
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getTestIter(JNIEnv* env, jobject self, jint idx) {
  return cos_net_get_test_iter(native(env, self), idx);
}
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getTestInterval(JNIEnv* env, jobject self) {
  return cos_net_get_test_interval(native(env, self));
}
JNIEXPORT jint JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_snapshot(JNIEnv* env, jobject self) {
  return cos_net_snapshot(native(env, self));
}

// ()[Ljava/lang/String; and (I)[Lcom/yahoo/ml/jcaffe/FloatBlob;   JniCaffeNet.cpp:587-673
JNIEXPORT jobjectArray JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getValidationOutputBlobNames(JNIEnv*, jobject) {
  return nullptr;
}
JNIEXPORT jobjectArray JNICALL Java_com_yahoo_ml_jcaffe_CaffeNet_getValidationOutputBlobs(JNIEnv*, jobject, jint) {
  return nullptr;
}

}  // extern "C"
#endif  // COS_HAVE_JNI
