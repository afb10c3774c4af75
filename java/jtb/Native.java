package jtb;

/**
 * JNI surface of the H100 history checker: one static native method per C-ABI entry point of libjtb_check.so
 * (include/jtb_check.h), implemented by jni/jtb_jni.c (libjtb_jni.so).  Used by clj/jtb/checker.clj.
 *
 * <p>A flattened history travels as ONE {@code Object[14]} of primitive arrays laid out like {@code struct
 * jtb_history}: {@code [byte[] type, byte[] f, byte[] flags, int[] process, int[] index, long[] timeNs, int[] a,
 * int[] b, int[] c, long[] payloadOff, int[] payloadLen, int[] payload, long[] shardOff, long[] keyIds]}.
 * Results come back as flat {@code long[]} / {@code int[]} records (layouts below) that the Clojure side turns into
 * the checker result maps.  A native error is a {@link RuntimeException}, so jepsen's {@code check-safe} reports
 * {@code {:valid? :unknown :error ...}} exactly as it does for a throwing Clojure checker.
 */
public final class Native {
    static {
        System.loadLibrary("jtb_jni");
    }

    private Native() {}

    /** {@code jtb_opts.flags} bits (include/jtb_check.h). */
    public static final int OPT_NO_EAGER_READS = 1, OPT_NO_SCOUTS = 2, OPT_ENGINE_LEVEL = 4, OPT_ENGINE_WORKLIST = 8,
            OPT_NO_BEAM = 16;

    /** Number of CUDA devices ({@code jtb_device_count}). */
    public static native int deviceCount();

    /** {@code jtb_create}: one context = one device + stream + cached buffers; calls on it are serialised. */
    public static native long create(int device, int flags, long tableBytes, long maxConfigs, int timeBudgetMs);

    public static native void destroy(long ctx);

    /** {@code jtb_multi_create}: in-library fan-out over nGpus devices (0 = all) with one NCCL all-reduce(MAX). */
    public static native long multiCreate(int nGpus, int flags, long tableBytes, long maxConfigs, int timeBudgetMs);

    public static native void multiDestroy(long multi);

    /**
     * {@code jtb_check_linearizable} (multi == false, handle from {@link #create}) or
     * {@code jtb_multi_check_linearizable} (multi == true, handle from {@link #multiCreate}).
     *
     * @return {@code [valid, nFailures, configs, probes, kernelNs, totalNs, keyBytes, nShards]} followed by 7 longs
     *     per shard: {@code valid, witnessIndex, previousOkIndex, cause, configs, probes, device}
     */
    public static native long[] checkLinearizable(long handle, boolean multi, Object[] history, int modelKind,
                                                  int initValue, int[] accounts, int[] initBalances, boolean negativeOk);

    /**
     * {@code jtb_final_configs}: knossos' {@code :configs} of an INVALID shard; call directly after
     * {@link #checkLinearizable} (multi == false) on the same history.
     *
     * @return {@code [total]} followed by min(cap, total) records of 140 ints in {@code jtb_final_config} field order
     */
    public static native int[] finalConfigs(long ctx, Object[] history, int modelKind, int initValue, int[] accounts,
                                            int[] initBalances, boolean negativeOk, int shard, int cap);

    /**
     * {@code jtb_check_set_full} / {@code jtb_multi_check_set_full} (per-shard structs only when multi).
     *
     * @return {@code [valid, nFailures, raiaValid, nSuspect, kernelNs, totalNs, nShards, nElems]}, then 10 longs per
     *     shard ({@code valid, attempt, stable, lost, neverRead, stale, duplicated, suspectFinalReads,
     *     stableLatencyMaxMs, lostLatencyMaxMs}), then {@code elemOff[nShards + 1]}, then 4 longs per element
     *     ({@code id, outcome, latencyMs, dupCount}), then per suspect final read {@code shard, index, nMissing,
     *     missing ids...}
     */
    public static native long[] checkSetFull(long handle, boolean multi, Object[] history, boolean linearizable);

    /**
     * {@code jtb_check_bank_totals}.
     *
     * @return {@code [valid, referenceThrows, readCount, errorCount, firstErrorIndex, firstErrorType, count[5],
     *     firstIndex[5], lastIndex[5], worstIndex[5], lowestTotal, highestTotal, lowestIndex, highestIndex, kernelNs,
     *     totalNs]} (34 longs)
     */
    public static native long[] checkBankTotals(long ctx, Object[] history, int[] accounts, long totalAmount,
                                                boolean negativeOk);

    /**
     * {@code jtb_check_monotonic_keys}: Elle's monotonic-key graph over the :ok reads, real-time edges unless
     * {@code realtime} is false.  Read payloads are (key, valueLo, valueHi) triples, key = 2 * account + field
     * (0 debits-posted, 1 credits-posted).
     *
     * @return {@code [valid, nFailures, nReads, kernelNs, totalNs, nShards]} followed by 14 longs per shard:
     *     {@code valid, cause, nReads, nKeys, witnessIndex, partnerIndex}, then for the edges partner -> witness and
     *     witness -> partner {@code kind, key, value, value'}
     */
    public static native long[] checkMonotonicKeys(long ctx, Object[] history, boolean realtime);

    /**
     * {@code jtb_check_counter_bounds}: every counter an :ok read observes against L (the :ok transfers completed
     * before the read was invoked) and U (the non-:fail transfers invoked before it completed).  Input as for
     * {@link #checkMonotonicKeys}; transfers carry amount, debit account and credit account in a, b, c.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nViolations, kernelNs, totalNs, nShards]} followed by 12
     *     longs per shard: {@code valid, nReads, nTransfers, nKeys, nBelow, nAbove, witnessIndex, witnessKey, kind,
     *     culpritIndex, value, bound}
     */
    public static native long[] checkCounterBounds(long ctx, Object[] history);

    /**
     * {@code jtb_check_transfer_lookups}: the transfer records :ok lookups return against the transfers clients issued
     * and the counters reads show.  Input: the ledger-lookups form (transfer invokes and :ok lookups carry records of
     * 5 ints: id lo, id hi, debit, credit, amount; lookups have f = 5).
     *
     * @return {@code [valid, nFailures, nLookups, nRecords, nTransfers, nReads, nViolations, kernelNs, totalNs,
     *     nShards]} followed by 21 longs per shard: {@code valid, nLookups, nRecords, nTransfers, nReads}, the 9 counts
     *     by kind, {@code witnessIndex, kind, transferId, key, relatedIndex, value, bound}
     */
    public static native long[] checkTransferLookups(long ctx, Object[] history);

    /**
     * {@code jtb_check_read_explanations}: whether one set of transfers explains every counter each :ok read shows.
     * Input: the ledger-lookups form.  {@code maxNodes <= 0} is the default per-read search budget.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nExplained, nUnexplained, nUndecided, nodes, kernelNs,
     *     totalNs, nShards]} followed by 15 longs per shard: {@code valid, nReads, nTransfers, witnessIndex,
     *     nExplained, nUndecided, nKey, nJoint, nodes, kind, key, nMust, nMay, value, mustSum}
     */
    public static native long[] checkReadExplanations(long ctx, Object[] history, long maxNodes);

    /**
     * {@code jtb_check_read_gaps}: whether the transfers committed between two successive :ok reads explain what
     * changed.  Input: the ledger-lookups form.  {@code maxNodes <= 0} is the default per-gap search budget.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nExplained, nUnexplained, nDouble, nUndecided, nodes,
     *     kernelNs, totalNs, nShards]} followed by 18 longs per shard: {@code valid, cause, nReads, nTransfers,
     *     nExplained, nUndecided, nKey, nJoint, nDouble, nodes, witnessIndex, lowerIndex, kind, key, delta,
     *     transferId, otherIndex, nEligible}
     */
    public static native long[] checkReadGaps(long ctx, Object[] history, long maxNodes);

    /**
     * {@code jtb_check_transfer_placement}: the read-gap check with located transfers carried across gaps to a
     * fixpoint.  Input: the ledger-lookups form.  {@code maxNodes <= 0} and {@code maxRounds <= 0} are the defaults.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nExplained, nUnexplained, nDouble, nLost, nUndecided,
     *     nPlaced, nodes, rounds, kernelNs, totalNs, nShards]} followed by 22 longs per shard: {@code valid, cause,
     *     nReads, nTransfers, nExplained, nUndecided, nKey, nJoint, nDouble, nLost, nPlaced, nodes, rounds,
     *     witnessIndex, lowerIndex, kind, key, round, delta, transferId, otherIndex, nEligible}
     */
    public static native long[] checkTransferPlacement(long ctx, Object[] history, long maxNodes, int maxRounds);

    /**
     * {@code jtb_check_serial_witness}: a proof that a ledger history is linearizable (VALID), or UNKNOWN with a
     * cause; never INVALID.  Input: the ledger-lookups form.  {@code maxNodes} and {@code maxRounds} as for
     * {@link #checkTransferPlacement}, which it runs first.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     kernelNs, totalNs, nShards]} followed by 11 longs per shard: {@code valid, cause, nReads, nTransfers,
     *     nCommitted, nCommittedCrashed, nAfter, nodes, rounds, failIndex, transferId}
     */
    public static native long[] checkSerialWitness(long ctx, Object[] history, long maxNodes, int maxRounds);

    /**
     * {@code jtb_check_repaired_witness}: {@link #checkSerialWitness} with up to {@code maxRepairs} repair rounds
     * (<= 0: the library's default) on the shards it leaves no-witness or real-time.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     repairs, nBans, kernelNs, totalNs, nShards]} followed by 13 longs per shard: {@code valid, cause, nReads,
     *     nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds, failIndex, transferId, repairs, nBans}
     */
    public static native long[] checkRepairedWitness(long ctx, Object[] history, long maxNodes, int maxRounds,
                                                     int maxRepairs);

    /**
     * {@code jtb_check_lifted_witness}: {@link #checkRepairedWitness} with up to {@code maxLifts} lift steps (<= 0: the
     * library's default) on the shards whose repairs stop because a repair recorded no new ban.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     repairs, nBans, lifts, nLifted, kernelNs, totalNs, nShards]} followed by 15 longs per shard: {@code valid,
     *     cause, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds, failIndex, transferId,
     *     repairs, nBans, lifts, nLifted}
     */
    public static native long[] checkLiftedWitness(long ctx, Object[] history, long maxNodes, int maxRounds,
                                                   int maxRepairs, int maxLifts);

    /**
     * {@code jtb_check_class_witness}: {@link #checkLiftedWitness}, then a class pass on the shards it leaves unknown
     * (undecided, no-witness or real-time), with the same budgets.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     repairs, nBans, lifts, nLifted, classRounds, nHanded, kernelNs, totalNs, nShards]} followed by 18 longs per
     *     shard: {@code valid, cause, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     failIndex, transferId, repairs, nBans, lifts, nLifted, classCause, classRounds, nHanded}
     */
    public static native long[] checkClassWitness(long ctx, Object[] history, long maxNodes, int maxRounds,
                                                  int maxRepairs, int maxLifts);

    /**
     * {@code jtb_check_lookup_witness}: {@link #checkClassWitness}, then every :ok lookup of a shard it proves placed
     * in the serial order, with the same budgets.
     *
     * @return {@code [valid, nFailures, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes, rounds,
     *     repairs, nBans, lifts, nLifted, classRounds, nHanded, nLookupsPlaced, kernelNs, totalNs, nShards]} followed
     *     by 21 longs per shard: {@code valid, cause, nReads, nTransfers, nCommitted, nCommittedCrashed, nAfter, nodes,
     *     rounds, failIndex, transferId, repairs, nBans, lifts, nLifted, classCause, classRounds, nHanded, lookupCause,
     *     lookupFailIndex, nLookupsPlaced}
     */
    public static native long[] checkLookupWitness(long ctx, Object[] history, long maxNodes, int maxRounds,
                                                   int maxRepairs, int maxLifts);
}
