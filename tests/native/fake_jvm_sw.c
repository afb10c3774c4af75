/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkSerialWitness (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkSerialWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                jobjectArray history, jlong max_nodes,
                                                                jint max_rounds);

void* fj_check_serial_witness(long long h, void* hist, long long max_nodes, int max_rounds) {
    return Java_jtb_Native_checkSerialWitness(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jlong)max_nodes,
                                              (jint)max_rounds);
}
