/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkReadGaps (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkReadGaps(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                           jlong max_nodes);

void* fj_check_read_gaps(long long h, void* hist, long long max_nodes) {
    return Java_jtb_Native_checkReadGaps(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jlong)max_nodes);
}
