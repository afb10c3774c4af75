/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkTransferPlacement (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkTransferPlacement(JNIEnv* env, jclass cls, jlong handle,
                                                                    jobjectArray history, jlong max_nodes,
                                                                    jint max_rounds);

void* fj_check_transfer_placement(long long h, void* hist, long long max_nodes, int max_rounds) {
    return Java_jtb_Native_checkTransferPlacement(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jlong)max_nodes,
                                                  (jint)max_rounds);
}
