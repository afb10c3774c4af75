/*
 * jtb_jni.c — JNI shim between jtb.Native (java/jtb/Native.java, used by clj/jtb/checker.clj) and the C ABI of
 * libjtb_check.so (include/jtb_check.h).  One exported function per `native` method of jtb.Native.
 *
 * Build on a host with a JDK (jni/Makefile):
 *     gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../include \
 *         jtb_jni.c -L../jepsen_tigerbeetle_b200 -ljtb_check -o libjtb_jni.so
 * This image has no JDK: here the file is compiled against jni/stub/jni.h and driven end to end by
 * tests/native/fake_jvm.c (a JNIEnv over plain C arrays) — tests/test_jni_shim.py.
 *
 * Pure marshalling.  Arrays are obtained with Get<Type>ArrayElements / released with JNI_ABORT (read-only), NOT with
 * GetPrimitiveArrayCritical: a search can run for seconds and a critical section would block the JVM's GC that long.
 * A non-zero status becomes a RuntimeException so that jepsen's check-safe yields {:valid? :unknown :error ...}
 * (SURVEY §8(b) error convention).
 */
#include <jni.h>
#include <stdlib.h>
#include <string.h>

#include "jtb_check.h"

static void throw_rt(JNIEnv* env, const char* msg) {
    jclass c = (*env)->FindClass(env, "java/lang/RuntimeException");
    if (c) (*env)->ThrowNew(env, c, msg);
}

/* ---- the flattened history: Object[14] of primitive arrays in `struct jtb_history` order ------------------- */
enum { H_TYPE, H_F, H_FLAGS, H_PROCESS, H_INDEX, H_TIME, H_A, H_B, H_C, H_POFF, H_PLEN, H_PAYLOAD, H_SOFF, H_KEYS, H_N };
static const char H_KIND[H_N] = {'b', 'b', 'b', 'i', 'i', 'l', 'i', 'i', 'i', 'l', 'i', 'i', 'l', 'l'};

typedef struct {
    jarray arr[H_N];
    void* ptr[H_N];
} hist_pins;

static void unpin_history(JNIEnv* env, hist_pins* p) {
    for (int i = 0; i < H_N; ++i) {
        if (!p->arr[i] || !p->ptr[i]) continue;
        if (H_KIND[i] == 'b') (*env)->ReleaseByteArrayElements(env, p->arr[i], (jbyte*)p->ptr[i], JNI_ABORT);
        else if (H_KIND[i] == 'i') (*env)->ReleaseIntArrayElements(env, p->arr[i], (jint*)p->ptr[i], JNI_ABORT);
        else (*env)->ReleaseLongArrayElements(env, p->arr[i], (jlong*)p->ptr[i], JNI_ABORT);
        p->ptr[i] = NULL;
    }
}

/* returns 0, or -1 with a pending RuntimeException */
static int pin_history(JNIEnv* env, jobjectArray hist, jtb_history* h, hist_pins* p) {
    memset(p, 0, sizeof *p);
    memset(h, 0, sizeof *h);
    if (!hist || (*env)->GetArrayLength(env, hist) != H_N) {
        throw_rt(env, "history must be an Object[14] of primitive arrays (see jtb.Native)");
        return -1;
    }
    for (int i = 0; i < H_N; ++i) {
        p->arr[i] = (jarray)(*env)->GetObjectArrayElement(env, hist, i);
        if (!p->arr[i]) {
            if (i == H_FLAGS || i == H_KEYS) continue; /* optional in the C ABI */
            unpin_history(env, p);
            throw_rt(env, "history array is null");
            return -1;
        }
        if (H_KIND[i] == 'b') p->ptr[i] = (*env)->GetByteArrayElements(env, p->arr[i], NULL);
        else if (H_KIND[i] == 'i') p->ptr[i] = (*env)->GetIntArrayElements(env, p->arr[i], NULL);
        else p->ptr[i] = (*env)->GetLongArrayElements(env, p->arr[i], NULL);
        if (!p->ptr[i]) {
            unpin_history(env, p);
            throw_rt(env, "out of memory pinning a history array");
            return -1;
        }
    }
    h->n_events = (*env)->GetArrayLength(env, p->arr[H_TYPE]);
    h->n_payload = (*env)->GetArrayLength(env, p->arr[H_PAYLOAD]);
    h->n_shards = (*env)->GetArrayLength(env, p->arr[H_SOFF]) - 1;
    h->type = (const uint8_t*)p->ptr[H_TYPE];
    h->f = (const uint8_t*)p->ptr[H_F];
    h->flags = (const uint8_t*)p->ptr[H_FLAGS];
    h->process = (const int32_t*)p->ptr[H_PROCESS];
    h->index = (const int32_t*)p->ptr[H_INDEX];
    h->time_ns = (const int64_t*)p->ptr[H_TIME];
    h->a = (const int32_t*)p->ptr[H_A];
    h->b = (const int32_t*)p->ptr[H_B];
    h->c = (const int32_t*)p->ptr[H_C];
    h->payload_off = (const int64_t*)p->ptr[H_POFF];
    h->payload_len = (const int32_t*)p->ptr[H_PLEN];
    h->payload = (const int32_t*)p->ptr[H_PAYLOAD];
    h->shard_off = (const int64_t*)p->ptr[H_SOFF];
    h->key_ids = (const int64_t*)p->ptr[H_KEYS];
    if (h->n_shards < 0) {
        unpin_history(env, p);
        throw_rt(env, "shardOff must have n_shards + 1 entries");
        return -1;
    }
    return 0;
}

static int fill_model(JNIEnv* env, jtb_model* m, jint kind, jint init_value, jintArray accounts, jintArray init_balances,
                      jboolean neg_ok) {
    memset(m, 0, sizeof *m);
    m->kind = kind;
    m->init_value = init_value;
    m->negative_balances_ok = neg_ok ? 1 : 0;
    if (accounts) {
        const jsize n = (*env)->GetArrayLength(env, accounts);
        if (n > JTB_MAX_ACCOUNTS) { throw_rt(env, "at most 8 accounts"); return -1; }
        m->n_accounts = n;
        (*env)->GetIntArrayRegion(env, accounts, 0, n, (jint*)m->account_ids);
        if (init_balances) {
            if ((*env)->GetArrayLength(env, init_balances) != n) { throw_rt(env, "initBalances must match accounts"); return -1; }
            (*env)->GetIntArrayRegion(env, init_balances, 0, n, (jint*)m->init_balance);
        }
    }
    return 0;
}

static void fill_opts(jtb_opts* o, jint device, jint flags, jlong table_bytes, jlong max_configs, jint time_budget_ms) {
    memset(o, 0, sizeof *o);
    o->device = device;
    o->flags = flags;
    o->table_bytes = (uint64_t)table_bytes;
    o->max_configs = (uint64_t)max_configs;
    o->time_budget_ms = (uint32_t)time_budget_ms;
}

static jlong ns_of(double seconds) { return (jlong)(seconds * 1e9); }

/* ---- lifecycle -------------------------------------------------------------------------------------------- */
JNIEXPORT jint JNICALL Java_jtb_Native_deviceCount(JNIEnv* env, jclass cls) {
    (void)env; (void)cls;
    return jtb_device_count();
}

JNIEXPORT jlong JNICALL Java_jtb_Native_create(JNIEnv* env, jclass cls, jint device, jint flags, jlong table_bytes,
                                               jlong max_configs, jint time_budget_ms) {
    (void)cls;
    jtb_opts o;
    fill_opts(&o, device, flags, table_bytes, max_configs, time_budget_ms);
    jtb_ctx* ctx = jtb_create(&o);
    if (!ctx) throw_rt(env, "jtb_create failed: no CUDA device (there is no CPU fallback)");
    return (jlong)(intptr_t)ctx;
}

JNIEXPORT void JNICALL Java_jtb_Native_destroy(JNIEnv* env, jclass cls, jlong h) {
    (void)env; (void)cls;
    jtb_destroy((jtb_ctx*)(intptr_t)h);
}

JNIEXPORT jlong JNICALL Java_jtb_Native_multiCreate(JNIEnv* env, jclass cls, jint n_gpus, jint flags, jlong table_bytes,
                                                    jlong max_configs, jint time_budget_ms) {
    (void)cls;
    jtb_opts o;
    fill_opts(&o, 0, flags, table_bytes, max_configs, time_budget_ms);
    jtb_multi* mg = jtb_multi_create(&o, n_gpus);
    if (!mg) throw_rt(env, jtb_multi_create_error());
    return (jlong)(intptr_t)mg;
}

JNIEXPORT void JNICALL Java_jtb_Native_multiDestroy(JNIEnv* env, jclass cls, jlong h) {
    (void)env; (void)cls;
    jtb_multi_destroy((jtb_multi*)(intptr_t)h);
}

/* ---- hot path A9 ------------------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkLinearizable(JNIEnv* env, jclass cls, jlong handle, jboolean multi,
                                                               jobjectArray history, jint model_kind, jint init_value,
                                                               jintArray accounts, jintArray init_balances,
                                                               jboolean neg_ok) {
    (void)cls;
    jtb_history hist;
    jtb_model m;
    hist_pins pins;
    if (fill_model(env, &m, model_kind, init_value, accounts, init_balances, neg_ok)) return NULL;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_lin_shard* shards = (jtb_lin_shard*)calloc((size_t)(ns > 0 ? ns : 1), sizeof *shards);
    int32_t* dev = (int32_t*)calloc((size_t)(ns > 0 ? ns : 1), sizeof *dev);
    jtb_lin_result res;
    memset(&res, 0, sizeof res);
    int rc;
    const char* err = NULL;
    if (multi) {
        rc = jtb_multi_check_linearizable((jtb_multi*)(intptr_t)handle, &hist, &m, shards, &res, dev);
        if (rc) err = jtb_multi_last_error((jtb_multi*)(intptr_t)handle);
    } else {
        rc = jtb_check_linearizable((jtb_ctx*)(intptr_t)handle, &hist, &m, shards, &res);
        if (rc) err = jtb_last_error((jtb_ctx*)(intptr_t)handle);
    }
    unpin_history(env, &pins);
    jlongArray out = NULL;
    if (rc != 0) {
        throw_rt(env, err);
    } else {
        out = (*env)->NewLongArray(env, 8 + 7 * ns);
        if (out) {
            const jlong head[8] = {res.valid, res.n_failures, (jlong)res.configs_explored, (jlong)res.probes,
                                   ns_of(res.seconds_kernel), ns_of(res.seconds_total), res.key_bytes, ns};
            (*env)->SetLongArrayRegion(env, out, 0, 8, head);
            for (int s = 0; s < ns; ++s) {
                const jlong v[7] = {shards[s].valid, shards[s].witness_index, shards[s].previous_ok_index, shards[s].cause,
                                    (jlong)shards[s].configs_explored, (jlong)shards[s].probes, dev[s]};
                (*env)->SetLongArrayRegion(env, out, 8 + 7 * s, 7, v);
            }
        }
    }
    free(shards);
    free(dev);
    return out;
}

/* knossos' :configs of an INVALID shard; directly after checkLinearizable (multi == false) on the same arrays */
JNIEXPORT jintArray JNICALL Java_jtb_Native_finalConfigs(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                         jint model_kind, jint init_value, jintArray accounts,
                                                         jintArray init_balances, jboolean neg_ok, jint shard, jint cap) {
    (void)cls;
    jtb_history hist;
    jtb_model m;
    hist_pins pins;
    if (cap < 0) cap = 0;
    if (fill_model(env, &m, model_kind, init_value, accounts, init_balances, neg_ok)) return NULL;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    jtb_final_config* buf = (jtb_final_config*)calloc((size_t)(cap > 0 ? cap : 1), sizeof *buf);
    int64_t total = 0;
    const int rc = jtb_final_configs((jtb_ctx*)(intptr_t)handle, &hist, &m, shard, buf, cap, &total);
    unpin_history(env, &pins);
    jintArray out = NULL;
    if (rc != 0) {
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
    } else {
        const jsize rec = (jsize)(sizeof(jtb_final_config) / 4);
        const jsize n = (jsize)(total < cap ? total : cap);
        out = (*env)->NewIntArray(env, 1 + n * rec);
        if (out) {
            const jint t = (jint)total;
            (*env)->SetIntArrayRegion(env, out, 0, 1, &t);
            if (n) (*env)->SetIntArrayRegion(env, out, 1, n * rec, (const jint*)buf);
        }
    }
    free(buf);
    return out;
}

/* ---- hot path A4 (+ A5 read-all-invoked-adds in the same pass) ---------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkSetFull(JNIEnv* env, jclass cls, jlong handle, jboolean multi,
                                                          jobjectArray history, jboolean linearizable) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    /* capacities: every :invoke :add may start a tracked element; every :final? op may be a suspect read */
    int64_t n_elem_cap = 1, n_final = 1;
    if (!multi) {
        for (int64_t e = 0; e < hist.n_events; ++e) {
            n_elem_cap += hist.f[e] == JTB_F_ADD && hist.type[e] == JTB_T_INVOKE;
            n_final += hist.flags && (hist.flags[e] & JTB_FLAG_FINAL);
        }
    }
    int64_t miss_cap = n_final * n_elem_cap;
    if (miss_cap > (1ll << 26)) miss_cap = 1ll << 26;
    jtb_setfull_out o;
    memset(&o, 0, sizeof o);
    o.shards = (jtb_setfull_shard*)calloc((size_t)(ns > 0 ? ns : 1), sizeof *o.shards);
    int32_t* dev = (int32_t*)calloc((size_t)(ns > 0 ? ns : 1), sizeof *dev);
    o.elem_off = (int64_t*)calloc((size_t)ns + 1, 8);
    if (!multi) {
        o.elem_capacity = n_elem_cap;
        o.elem_id = (int32_t*)calloc((size_t)n_elem_cap, 4);
        o.elem_outcome = (uint8_t*)calloc((size_t)n_elem_cap, 1);
        o.elem_latency_ms = (int64_t*)calloc((size_t)n_elem_cap, 8);
        o.elem_dup_count = (int32_t*)calloc((size_t)n_elem_cap, 4);
        o.suspect_capacity = n_final;
        o.suspect_shard = (int32_t*)calloc((size_t)n_final, 4);
        o.suspect_index = (int32_t*)calloc((size_t)n_final, 4);
        o.suspect_missing_off = (int64_t*)calloc((size_t)n_final + 1, 8);
        o.missing_capacity = miss_cap;
        o.missing_ids = (int32_t*)calloc((size_t)miss_cap, 4);
    }
    int rc;
    const char* err = NULL;
    if (multi) {
        rc = jtb_multi_check_set_full((jtb_multi*)(intptr_t)handle, &hist, linearizable ? 1 : 0, &o, dev);
        if (rc) err = jtb_multi_last_error((jtb_multi*)(intptr_t)handle);
    } else {
        rc = jtb_check_set_full((jtb_ctx*)(intptr_t)handle, &hist, linearizable ? 1 : 0, &o);
        if (rc) err = jtb_last_error((jtb_ctx*)(intptr_t)handle);
    }
    unpin_history(env, &pins);
    jlongArray out = NULL;
    if (rc != 0) {
        throw_rt(env, err);
    } else {
        const int64_t n_elems = multi ? 0 : o.elem_off[ns];
        const int64_t n_sus = multi ? 0 : (o.n_suspect < o.suspect_capacity ? o.n_suspect : o.suspect_capacity);
        const int64_t n_miss = n_sus ? o.suspect_missing_off[n_sus] : 0;
        const int64_t total = 8 + 10ll * ns + (ns + 1) + 4 * n_elems + 3 * n_sus + n_miss;
        jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
        int64_t k = 0;
        v[k++] = o.valid; v[k++] = o.n_failures; v[k++] = o.raia_valid; v[k++] = o.n_suspect;
        v[k++] = ns_of(o.seconds_kernel); v[k++] = ns_of(o.seconds_total); v[k++] = ns; v[k++] = n_elems;
        for (int s = 0; s < ns; ++s) {
            const jtb_setfull_shard* q = &o.shards[s];
            v[k++] = q->valid; v[k++] = q->attempt_count; v[k++] = q->stable_count; v[k++] = q->lost_count;
            v[k++] = q->never_read_count; v[k++] = q->stale_count; v[k++] = q->duplicated_count;
            v[k++] = q->suspect_final_reads; v[k++] = q->stable_latency_max_ms; v[k++] = q->lost_latency_max_ms;
        }
        for (int s = 0; s <= ns; ++s) v[k++] = multi ? 0 : o.elem_off[s];
        for (int64_t e = 0; e < n_elems; ++e) {
            v[k++] = o.elem_id[e]; v[k++] = o.elem_outcome[e]; v[k++] = o.elem_latency_ms[e]; v[k++] = o.elem_dup_count[e];
        }
        for (int64_t i = 0; i < n_sus; ++i) {
            const int64_t lo = o.suspect_missing_off[i], hi = o.suspect_missing_off[i + 1];
            v[k++] = o.suspect_shard[i]; v[k++] = o.suspect_index[i]; v[k++] = hi - lo;
            for (int64_t j = lo; j < hi; ++j) v[k++] = o.missing_ids[j];
        }
        out = (*env)->NewLongArray(env, (jsize)k);
        if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
        free(v);
    }
    free(o.shards); free(dev); free(o.elem_off); free(o.elem_id); free(o.elem_outcome); free(o.elem_latency_ms);
    free(o.elem_dup_count); free(o.suspect_shard); free(o.suspect_index); free(o.suspect_missing_off); free(o.missing_ids);
    return out;
}

/* ---- hot path A8 ------------------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkBankTotals(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                             jintArray accounts, jlong total_amount, jboolean neg_ok) {
    (void)cls;
    jtb_history hist;
    jtb_model m;
    hist_pins pins;
    if (fill_model(env, &m, JTB_MODEL_BANK, 0, accounts, NULL, neg_ok)) return NULL;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    jtb_bank_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_bank_totals((jtb_ctx*)(intptr_t)handle, &hist, &m, total_amount, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    jlong v[34];
    int k = 0;
    v[k++] = r.valid; v[k++] = r.reference_throws; v[k++] = r.read_count; v[k++] = r.error_count;
    v[k++] = r.first_error_index; v[k++] = r.first_error_type;
    for (int t = 0; t < 5; ++t) v[k++] = r.count_by_type[t];
    for (int t = 0; t < 5; ++t) v[k++] = r.first_index_by_type[t];
    for (int t = 0; t < 5; ++t) v[k++] = r.last_index_by_type[t];
    for (int t = 0; t < 5; ++t) v[k++] = r.worst_index_by_type[t];
    v[k++] = r.lowest_total; v[k++] = r.highest_total; v[k++] = r.lowest_index; v[k++] = r.highest_index;
    v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total);
    jlongArray out = (*env)->NewLongArray(env, k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, k, v);
    return out;
}

/* ---- K7: monotonic-key check ------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkMonotonicKeys(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                                jboolean realtime) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_mono_shard* shards = (jtb_mono_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_mono_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_monotonic_keys((jtb_ctx*)(intptr_t)handle, &hist, realtime ? 0 : JTB_MONO_NO_REALTIME,
                                            shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 6 + 14ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = ns_of(r.seconds_kernel);
    v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_mono_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_keys; v[k++] = q->witness_index;
        v[k++] = q->partner_index;
        for (int e = 0; e < 2; ++e) {
            v[k++] = q->edge_kind[e]; v[k++] = q->edge_key[e]; v[k++] = q->edge_value[e]; v[k++] = q->edge_value2[e];
        }
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K8: counter-bounds check -------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkCounterBounds(JNIEnv* env, jclass cls, jlong handle, jobjectArray history) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_cb_shard* shards = (jtb_cb_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_cb_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_counter_bounds((jtb_ctx*)(intptr_t)handle, &hist, 0, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 8 + 12ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_violations;
    v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_cb_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_keys; v[k++] = q->n_below;
        v[k++] = q->n_above; v[k++] = q->witness_index; v[k++] = q->witness_key; v[k++] = q->kind;
        v[k++] = q->culprit_index; v[k++] = q->value; v[k++] = q->bound;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K9: transfer-lookup check ------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkTransferLookups(JNIEnv* env, jclass cls, jlong handle,
                                                                   jobjectArray history) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_tl_shard* shards = (jtb_tl_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_tl_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_transfer_lookups((jtb_ctx*)(intptr_t)handle, &hist, 0, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t per = 12 + JTB_TL_KINDS;
    const int64_t total = 10 + per * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_lookups; v[k++] = r.n_records; v[k++] = r.n_transfers;
    v[k++] = r.n_reads; v[k++] = r.n_violations; v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total);
    v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_tl_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->n_lookups; v[k++] = q->n_records; v[k++] = q->n_transfers; v[k++] = q->n_reads;
        for (int j = 0; j < JTB_TL_KINDS; ++j) v[k++] = q->count_by_kind[j];
        v[k++] = q->witness_index; v[k++] = q->kind; v[k++] = q->transfer_id; v[k++] = q->key;
        v[k++] = q->related_index; v[k++] = q->value; v[k++] = q->bound;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K10: read-explanation check ----------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkReadExplanations(JNIEnv* env, jclass cls, jlong handle,
                                                                    jobjectArray history, jlong max_nodes) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_rx_shard* shards = (jtb_rx_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_rx_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_read_explanations((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes, 0, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 11 + 15ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_explained;
    v[k++] = r.n_unexplained; v[k++] = r.n_undecided; v[k++] = r.nodes; v[k++] = ns_of(r.seconds_kernel);
    v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_rx_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->witness_index;
        v[k++] = q->n_explained; v[k++] = q->n_undecided; v[k++] = q->count_by_kind[0]; v[k++] = q->count_by_kind[1];
        v[k++] = q->nodes; v[k++] = q->kind; v[k++] = q->key; v[k++] = q->n_must; v[k++] = q->n_may;
        v[k++] = q->value; v[k++] = q->must_sum;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K11: read-gap check ------------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkReadGaps(JNIEnv* env, jclass cls, jlong handle, jobjectArray history,
                                                           jlong max_nodes) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_rg_shard* shards = (jtb_rg_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_rg_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_read_gaps((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes, 0, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 12 + 18ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_explained;
    v[k++] = r.n_unexplained; v[k++] = r.n_double; v[k++] = r.n_undecided; v[k++] = r.nodes;
    v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_rg_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_explained;
        v[k++] = q->n_undecided; v[k++] = q->count_by_kind[0]; v[k++] = q->count_by_kind[1];
        v[k++] = q->count_by_kind[2]; v[k++] = q->nodes; v[k++] = q->witness_index; v[k++] = q->lower_index;
        v[k++] = q->kind; v[k++] = q->key; v[k++] = q->delta; v[k++] = q->transfer_id; v[k++] = q->other_index;
        v[k++] = q->n_eligible;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K12: transfer-placement check ------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkTransferPlacement(JNIEnv* env, jclass cls, jlong handle,
                                                                    jobjectArray history, jlong max_nodes,
                                                                    jint max_rounds) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_tp_shard* shards = (jtb_tp_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_tp_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_transfer_placement((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes,
                                                (int32_t)max_rounds, 0, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 15 + 22ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_explained;
    v[k++] = r.n_unexplained; v[k++] = r.n_double; v[k++] = r.n_lost; v[k++] = r.n_undecided; v[k++] = r.n_placed;
    v[k++] = r.nodes; v[k++] = r.rounds; v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total);
    v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_tp_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_explained;
        v[k++] = q->n_undecided; v[k++] = q->count_by_kind[0]; v[k++] = q->count_by_kind[1];
        v[k++] = q->count_by_kind[2]; v[k++] = q->count_by_kind[3]; v[k++] = q->n_placed; v[k++] = q->nodes;
        v[k++] = q->rounds; v[k++] = q->witness_index; v[k++] = q->lower_index; v[k++] = q->kind; v[k++] = q->key;
        v[k++] = q->round; v[k++] = q->delta; v[k++] = q->transfer_id; v[k++] = q->other_index;
        v[k++] = q->n_eligible;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K13: serial-witness check --------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkSerialWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                jobjectArray history, jlong max_nodes,
                                                                jint max_rounds) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_sw_shard* shards = (jtb_sw_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_sw_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_serial_witness((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes,
                                            (int32_t)max_rounds, 0, NULL, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 12 + 11ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_committed;
    v[k++] = r.n_committed_crashed; v[k++] = r.n_after; v[k++] = r.nodes; v[k++] = r.rounds;
    v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_sw_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_committed;
        v[k++] = q->n_committed_crashed; v[k++] = q->n_after; v[k++] = q->nodes; v[k++] = q->rounds;
        v[k++] = q->fail_index; v[k++] = q->transfer_id;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K14: repaired serial witness ------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkRepairedWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                  jobjectArray history, jlong max_nodes,
                                                                  jint max_rounds, jint max_repairs) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_rw_shard* shards = (jtb_rw_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_rw_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_repaired_witness((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes,
                                              (int32_t)max_rounds, (int32_t)max_repairs, 0, NULL, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 14 + 13ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_committed;
    v[k++] = r.n_committed_crashed; v[k++] = r.n_after; v[k++] = r.nodes; v[k++] = r.rounds; v[k++] = r.repairs;
    v[k++] = r.n_bans; v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_rw_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_committed;
        v[k++] = q->n_committed_crashed; v[k++] = q->n_after; v[k++] = q->nodes; v[k++] = q->rounds;
        v[k++] = q->fail_index; v[k++] = q->transfer_id; v[k++] = q->repairs; v[k++] = q->n_bans;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K15: lifted serial witness -------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkLiftedWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                jobjectArray history, jlong max_nodes, jint max_rounds,
                                                                jint max_repairs, jint max_lifts) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_lw_shard* shards = (jtb_lw_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_lw_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_lifted_witness((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes, (int32_t)max_rounds,
                                            (int32_t)max_repairs, (int32_t)max_lifts, 0, NULL, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 16 + 15ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_committed;
    v[k++] = r.n_committed_crashed; v[k++] = r.n_after; v[k++] = r.nodes; v[k++] = r.rounds; v[k++] = r.repairs;
    v[k++] = r.n_bans; v[k++] = r.lifts; v[k++] = r.n_lifted; v[k++] = ns_of(r.seconds_kernel);
    v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_lw_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_committed;
        v[k++] = q->n_committed_crashed; v[k++] = q->n_after; v[k++] = q->nodes; v[k++] = q->rounds;
        v[k++] = q->fail_index; v[k++] = q->transfer_id; v[k++] = q->repairs; v[k++] = q->n_bans; v[k++] = q->lifts;
        v[k++] = q->n_lifted;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K16: class witness ------------------------------------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkClassWitness(JNIEnv* env, jclass cls, jlong handle,
                                                               jobjectArray history, jlong max_nodes, jint max_rounds,
                                                               jint max_repairs, jint max_lifts) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_cw_shard* shards = (jtb_cw_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_cw_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_class_witness((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes, (int32_t)max_rounds,
                                           (int32_t)max_repairs, (int32_t)max_lifts, 0, NULL, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 18 + 18ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_committed;
    v[k++] = r.n_committed_crashed; v[k++] = r.n_after; v[k++] = r.nodes; v[k++] = r.rounds; v[k++] = r.repairs;
    v[k++] = r.n_bans; v[k++] = r.lifts; v[k++] = r.n_lifted; v[k++] = r.class_rounds; v[k++] = r.n_handed;
    v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_cw_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_committed;
        v[k++] = q->n_committed_crashed; v[k++] = q->n_after; v[k++] = q->nodes; v[k++] = q->rounds;
        v[k++] = q->fail_index; v[k++] = q->transfer_id; v[k++] = q->repairs; v[k++] = q->n_bans; v[k++] = q->lifts;
        v[k++] = q->n_lifted; v[k++] = q->class_cause; v[k++] = q->class_rounds; v[k++] = q->n_handed;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}

/* ---- K17: lookup witness ----------------------------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_jtb_Native_checkLookupWitness(JNIEnv* env, jclass cls, jlong handle,
                                                                jobjectArray history, jlong max_nodes, jint max_rounds,
                                                                jint max_repairs, jint max_lifts) {
    (void)cls;
    jtb_history hist;
    hist_pins pins;
    if (pin_history(env, history, &hist, &pins)) return NULL;
    const int ns = hist.n_shards;
    jtb_lk_shard* shards = (jtb_lk_shard*)calloc(ns > 0 ? (size_t)ns : 1, sizeof *shards);
    jtb_lk_result r;
    memset(&r, 0, sizeof r);
    const int rc = jtb_check_lookup_witness((jtb_ctx*)(intptr_t)handle, &hist, (int64_t)max_nodes,
                                            (int32_t)max_rounds, (int32_t)max_repairs, (int32_t)max_lifts, 0, NULL,
                                            NULL, shards, &r);
    unpin_history(env, &pins);
    if (rc != 0) {
        free(shards);
        throw_rt(env, jtb_last_error((jtb_ctx*)(intptr_t)handle));
        return NULL;
    }
    const int64_t total = 19 + 21ll * ns;
    jlong* v = (jlong*)calloc((size_t)total, sizeof *v);
    int64_t k = 0;
    v[k++] = r.valid; v[k++] = r.n_failures; v[k++] = r.n_reads; v[k++] = r.n_transfers; v[k++] = r.n_committed;
    v[k++] = r.n_committed_crashed; v[k++] = r.n_after; v[k++] = r.nodes; v[k++] = r.rounds; v[k++] = r.repairs;
    v[k++] = r.n_bans; v[k++] = r.lifts; v[k++] = r.n_lifted; v[k++] = r.class_rounds; v[k++] = r.n_handed;
    v[k++] = r.n_lookups_placed; v[k++] = ns_of(r.seconds_kernel); v[k++] = ns_of(r.seconds_total); v[k++] = ns;
    for (int s = 0; s < ns; ++s) {
        const jtb_lk_shard* q = &shards[s];
        v[k++] = q->valid; v[k++] = q->cause; v[k++] = q->n_reads; v[k++] = q->n_transfers; v[k++] = q->n_committed;
        v[k++] = q->n_committed_crashed; v[k++] = q->n_after; v[k++] = q->nodes; v[k++] = q->rounds;
        v[k++] = q->fail_index; v[k++] = q->transfer_id; v[k++] = q->repairs; v[k++] = q->n_bans; v[k++] = q->lifts;
        v[k++] = q->n_lifted; v[k++] = q->class_cause; v[k++] = q->class_rounds; v[k++] = q->n_handed;
        v[k++] = q->lookup_cause; v[k++] = q->lookup_fail_index; v[k++] = q->n_lookups_placed;
    }
    jlongArray out = (*env)->NewLongArray(env, (jsize)k);
    if (out) (*env)->SetLongArrayRegion(env, out, 0, (jsize)k, v);
    free(v);
    free(shards);
    return out;
}
