/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkRepairedWitness (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkRepairedWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                  jobjectArray history, jlong max_nodes,
                                                                  jint max_rounds, jint max_repairs);

void* fj_check_repaired_witness(long long h, void* hist, long long max_nodes, int max_rounds, int max_repairs) {
    return Java_jtb_Native_checkRepairedWitness(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jlong)max_nodes,
                                                (jint)max_rounds, (jint)max_repairs);
}
