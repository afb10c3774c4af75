/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkCounterBounds (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkCounterBounds(JNIEnv* env, jclass cls, jlong handle, jobjectArray history);

void* fj_check_counter_bounds(long long h, void* hist) {
    return Java_jtb_Native_checkCounterBounds(&g_env, NULL, (jlong)h, (jobjectArray)hist);
}
