/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkTransferLookups (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkTransferLookups(JNIEnv* env, jclass cls, jlong handle,
                                                                   jobjectArray history);

void* fj_check_transfer_lookups(long long h, void* hist) {
    return Java_jtb_Native_checkTransferLookups(&g_env, NULL, (jlong)h, (jobjectArray)hist);
}
