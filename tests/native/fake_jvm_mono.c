/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkMonotonicKeys (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkMonotonicKeys(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                                jboolean realtime);

void* fj_check_monotonic_keys(long long h, void* hist, int realtime) {
    return Java_jtb_Native_checkMonotonicKeys(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jboolean)realtime);
}
