/* The fake JVM of fake_jvm.c plus a driver for jtb.Native.checkLookupWitness (TEST INFRASTRUCTURE). */
#include "fake_jvm.c"

JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkLookupWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                jobjectArray history, jlong max_nodes, jint max_rounds,
                                                                jint max_repairs, jint max_lifts);

void* fj_check_lookup_witness(long long h, void* hist, long long max_nodes, int max_rounds, int max_repairs,
                              int max_lifts) {
    return Java_jtb_Native_checkLookupWitness(&g_env, NULL, (jlong)h, (jobjectArray)hist, (jlong)max_nodes,
                                              (jint)max_rounds, (jint)max_repairs, (jint)max_lifts);
}
