(ns jtb.checker
  "Clojure glue for the H100 history checker: jepsen.checker/Checker implementations that flatten the history, call
  libjtb_check.so through jtb.Native (java/jtb/Native.java -> jni/jtb_jni.c) and build the SAME result maps the
  reference's checkers return.

  This image has no JVM/Clojure: the file cannot be loaded here.  What IS checked here (tests/test_jni_shim.py):
  every Native/<method> call below exists in jtb/Native.java with that arity, every native method has its
  Java_jtb_Native_<method> export in jni/jtb_jni.c, and the shim itself runs end to end against the library through
  a fake JNIEnv.  The tested twin of the map-building below is jepsen_tigerbeetle_b200/{history,checker}.py.

  Drop-in use in the reference (nurturenature/jepsen-tigerbeetle):

    ;; src/tigerbeetle/workloads/set_full.clj:155-158
    :checker (jtb/independent-checker                                           ; was independent/checker + compose
              {:set-full              [:set-full {:linearizable? true}]         ; was checker/set-full
               :linear                [:linearizable {:model :set}]             ; new, optional
               :read-all-invoked-adds [:read-all-invoked-adds]})                ; was (read-all-invoked-adds)
    ;; or, keeping jepsen's own fan-out (one native call per key):
    :checker (independent/checker
              (checker/compose {:set-full              (jtb/set-full {:linearizable? true})
                                :read-all-invoked-adds (jtb/read-all-invoked-adds)}))

    ;; src/tigerbeetle/tests/ledger.clj:363-367
    :checker (checker/compose
              {:SI     (jtb/bank-checker checker-opts)                          ; was (checker checker-opts)
               :linear (jtb/linearizable {:model :bank})                        ; new
               ...})"
  (:require [jepsen.checker :as checker]
            [jepsen.independent :as independent])
  (:import (jtb Native)))

;; ---- codes (include/jtb_check.h) ---------------------------------------------------------------------------
(def type-code  {:invoke 0 :ok 1 :fail 2 :info 3})
(def f-code     {:read 0 :write 1 :cas 2 :add 3 :transfer 4 :lookup 5})
(def model-code {:register 0 :cas-register 1 :set 2 :bank 3})
(def NIL Integer/MIN_VALUE)
(def verdict    {0 true 1 :unknown 2 false})
(def cause      {0 nil 1 :table-full 2 :budget 3 :too-wide 4 :partial-read})
(def bank-error {1 :unexpected-key 2 :nil-balance 3 :wrong-total 4 :negative-value})

(defn- ledger->bank-op
  "tests/ledger.clj:89-114 for one client op; nil for :l-t ops (dropped there too)."
  [{:keys [type value] :as op}]
  (let [[f _ _] (first value)]
    (case f
      :r   (if (= :ok type)
             (assoc op :f :read
                    :value (reduce (fn [m [_ id {:keys [debits-posted credits-posted]}]]
                                     (assoc m id (- credits-posted debits-posted)))
                                   {} value))
             (assoc op :f :read :value nil))
      :t   (let [[_ _ v] (first value)] (assoc op :f :transfer :value v))
      :l-t nil
      nil)))

(defn- ledger->counters-op
  "One client op for the monotonic-key check: an :ok :r keeps every account's two counters as [key value-lo value-hi]
  triples, key = 2*account + field (0 debits-posted, 1 credits-posted); an account with nil amounts is left out (the
  read is then partial).  nil for :l-t ops, as ledger->bank drops them."
  [{:keys [type value] :as op}]
  (let [[f _ _] (first value)]
    (case f
      :r   (assoc op :f :read
                  :value (when (= :ok type)
                           (vec (for [[_ id amounts] value
                                      :when amounts
                                      :let [_ (when-not (and (<= 0 id) (< id (bit-shift-left 1 30)))
                                                (throw (IllegalArgumentException. (str "account " id " outside [0, 2^30)"))))]
                                      [field k] [[0 :debits-posted] [1 :credits-posted]]
                                      :let [x (get amounts k)]
                                      :when (some? x)
                                      :let [x (long x)]]
                                  [(+ (* 2 id) field) (unchecked-int x) (unchecked-int (bit-shift-right x 32))]))))
      :t   (let [[_ _ v] (first value)] (assoc op :f :transfer :value v))
      :l-t nil
      nil)))

(defn- transfer-records
  "[:t id {...}] / [:l-t id {...}] micro-ops -> [id-lo id-hi debit credit amount ...]; a lookup micro-op without a
  transfer map (not found) is left out."
  [value]
  (vec (for [[_ id v] value
             :when v
             x [(unchecked-int (long id)) (unchecked-int (bit-shift-right (long id) 32))
                (:debit-acct v) (:credit-acct v) (:amount v)]]
         x)))

(defn- ledger->lookups-ops
  "The ledger-lookups form of the client ops: ledger->counters-op, plus the records of a transfer invoke's [:t ...]
  micro-ops (all of them) in ::records, and every [:l-t ...] op as :f :lookup with its :ok records as :value.  An
  :ok lookup with an empty value takes its tag from its process's pending invoke."
  [ops]
  (first
    (reduce (fn [[out pending] {:keys [type value process f] :as op}]
              (if (not= :txn f)
                [(conj out op) pending]
                (let [tag     (or (ffirst value) (get pending process))
                      pending (if (= :invoke type) (assoc pending process tag) (dissoc pending process))
                      o       (case tag
                                :l-t (assoc op :f :lookup :value (when (= :ok type) (transfer-records value)))
                                :t   (cond-> (ledger->counters-op op)
                                       (= :invoke type) (assoc ::records (transfer-records value)))
                                (ledger->counters-op op))]
                  [(if o (conj out o) out) pending])))
            [[] {}] ops)))

(defn- int-or-nil [x] (if (nil? x) NIL (int x)))

(defn flatten-history
  "history (seq of op maps) -> {:arrays Object[14] laid out as `struct jtb_history`, :keys [k ...], :by-index {idx op}}.
  Client ops only ((int? process)); independent tuples become CSR shards sorted by key; an op whose :value is a
  [nil nil] tuple (set_full.clj:112-116 with a rejected account creation) is skipped, like an element that was never
  tracked."
  [model history]
  (let [ops   (->> history (filter (comp int? :process)))
        ops   (->> (if (= model :ledger-lookups)
                     (ledger->lookups-ops ops)
                     (keep (fn [op] (if (= :txn (:f op))
                                      ((if (= model :ledger-counters) ledger->counters-op ledger->bank-op) op)
                                      op))
                           ops))
                   (keep (fn [op]
                           (let [v (:value op)]
                             (if (independent/tuple? v)
                               (when-not (nil? (key v)) (assoc op ::key (key v) :value (val v)))
                               (assoc op ::key nil))))))
        ks    (->> ops (map ::key) distinct (sort-by #(or % Long/MIN_VALUE)) vec)
        by-k  (group-by ::key ops)
        ops   (vec (mapcat by-k ks))
        n     (count ops)
        type  (byte-array n) f (byte-array n) flags (byte-array n)
        proc  (int-array n) index (int-array n) time (long-array n)
        a     (int-array n) b (int-array n) c (int-array n)
        poff  (long-array n) plen (int-array n)
        payload (java.util.ArrayList.)]
    (dotimes [i n]
      (let [o     (nth ops i)
            value (:value o)
            put-payload! (fn [xs]
                           (aset poff i (long (.size payload)))
                           (if (nil? xs)
                             (aset plen i (int -1))
                             (do (aset plen i (int (count xs)))
                                 (doseq [x xs] (.add payload (int x))))))]
        (aset ^bytes type i (byte (type-code (:type o))))
        (aset ^bytes f i (byte (get f-code (:f o) 0)))
        (aset ^bytes flags i (byte (if (:final? o) 1 0)))
        (aset proc i (int (:process o)))
        (aset index i (int (:index o)))
        (aset ^longs time i (long (or (:time o) 0)))
        (put-payload! nil)
        (case [model (:f o)]
          ([:register :read] [:cas-register :read])   (aset a i (int-or-nil value))
          ([:register :write] [:cas-register :write]) (aset a i (int-or-nil value))
          [:cas-register :cas] (do (aset a i (int-or-nil (first value))) (aset b i (int-or-nil (second value))))
          [:set :add]   (aset a i (int-or-nil value))
          [:set :read]  (put-payload! (when (and value (= :ok (:type o))) (sort value)))
          [:bank :read] (put-payload! (when (and value (= :ok (:type o)))
                                        (mapcat (fn [[id bal]] [id (int-or-nil bal)]) value)))
          ([:ledger-counters :read] [:ledger-lookups :read])
                            (put-payload! (when (and value (= :ok (:type o))) (apply concat value)))
          ([:bank :transfer] [:ledger-counters :transfer] [:ledger-lookups :transfer])
                            (do (aset a i (int (:amount value)))
                                (aset b i (int (or (:debit-acct value) (:from value))))
                                (aset c i (int (or (:credit-acct value) (:to value))))
                                (put-payload! (::records o)))
          [:ledger-lookups :lookup] (put-payload! value)
          nil)))                                    ; any other :f: opcode 0 with no value — ignored by every checker
    {:arrays   (object-array [type f flags proc index time a b c poff plen (int-array payload)
                              (long-array (reductions + 0 (map (comp count by-k) ks)))
                              (long-array (map #(if (integer? %) (long %) -1) ks))])
     :keys     ks
     :by-index (into {} (map (juxt :index identity)) history)}))

;; ---- contexts -----------------------------------------------------------------------------------------------
;; checker/compose and independent/checker call `check` from several threads; a context serialises its calls, so
;; one context per device is enough (jtb_ctx holds a mutex).  `*n-gpus*` > 1 selects the in-library fan-out
;; (jtb_multi_*: shards partitioned over the GPUs, one NCCL all-reduce(MAX) of the verdict vector).
(def ^:dynamic *n-gpus* 1)
;; jtb_opts.flags (include/jtb_check.h, Native/OPT_*): 0 = defaults — eager reads, engine chosen from the history (level
;; engine for exhaustive sweeps, work list + beam + scouts for histories with crashed ops).  Rebind before first use, e.g.
;; (bit-or Native/OPT_NO_EAGER_READS Native/OPT_ENGINE_LEVEL) to sweep exactly the configurations Knossos would visit.
(def ^:dynamic *flags* 0)
(defonce ^:private ctx   (delay (Native/create 0 (int *flags*) 0 0 0)))
(defonce ^:private multi (delay (Native/multiCreate 0 (int *flags*) 0 0 0)))
(defn- handle [] (if (> *n-gpus* 1) [@multi true] [@ctx false]))

(defn- model-args [model test]
  (let [accounts (vec (:accounts test (range 1 9)))]
    [(int (model-code model))
     (int-or-nil (:init-value test))
     (int-array accounts)
     (int-array (map #(get (:initial-balances test) % 0) accounts))
     (boolean (:negative-balances? test true))]))

;; ---- linearizable ---------------------------------------------------------------------------------------------
(defn- decode-configs
  "int[] from Native/finalConfigs -> [{:model .. :pending [{:index i} ..] ..}] (jtb_final_config is 140 ints)"
  [model accounts ^ints xs]
  (vec (for [off (range 1 (alength xs) 140)
             :let [rec (vec (java.util.Arrays/copyOfRange xs (int off) (int (+ off 140))))
                   np  (rec 9) nl (rec 10)]]
         {:model              (case model
                                :bank (zipmap accounts (subvec rec 1 9))
                                :set  nil
                                (let [s (rec 0)] (when-not (= s NIL) s)))
          :pending            (mapv #(hash-map :index %) (subvec rec 12 (+ 12 np)))
          :linearized-open    (mapv #(hash-map :index %) (subvec rec 76 (+ 76 nl)))
          :crashed-linearized (rec 11)})))

(defn- lin-shard-map
  "7 longs of one shard (valid witness previous-ok cause configs probes device) -> knossos-style analysis map"
  [by-index [valid witness prev cause-code configs _probes device]]
  (cond-> {:valid? (verdict valid) :analyzer :wgl-gpu :configs-explored configs :device device}
    (= 2 valid) (assoc :op (by-index witness) :previous-ok (when (<= 0 prev) (by-index prev)))
    (= 1 valid) (assoc :cause (cause cause-code))))

(defn- check-linearizable* [model test history]
  (let [{:keys [arrays keys by-index]} (flatten-history model history)
        [h multi?] (handle)
        [kind init accounts balances neg-ok] (model-args model test)
        res    (Native/checkLinearizable h multi? arrays kind init accounts balances neg-ok)
        shards (mapv #(lin-shard-map by-index %) (partition 7 (drop 8 res)))
        ;; knossos' :configs (first 10, like jepsen.checker/linearizable keeps them) for INVALID shards; the visited
        ;; table of the search is read, so: single context only, straight after the search, before any other call
        shards (if multi?
                 shards
                 (vec (map-indexed
                       (fn [s m]
                         (if (false? (:valid? m))
                           (let [xs (Native/finalConfigs h arrays kind init accounts balances neg-ok (int s) (int 10))]
                             (assoc m :configs (decode-configs model (vec accounts) xs) :configs-total (aget xs 0)))
                           m))
                       shards)))]
    {:keys keys :shards shards}))

(defn linearizable
  "Replacement for (checker/linearizable {:model m}); m in #{:register :cas-register :set :bank}."
  [{:keys [model]}]
  (assert model "The linearizable checker requires a model")
  (reify checker/Checker
    (check [_ test history _opts]
      (first (:shards (check-linearizable* model test history))))))

;; ---- set-full + read-all-invoked-adds -----------------------------------------------------------------------
(defn- quantiles [xs]
  (let [xs (vec (sort xs)) n (count xs)]
    (when (pos? n)
      (into {} (for [p [0 0.5 0.95 0.99 1]] [p (nth xs (min (dec n) (long (Math/floor (* n p)))))])))))

(defn- set-full-maps
  "long[] of Native/checkSetFull -> {:per-shard [set-full result map ...] :suspects {shard [[index missing] ...]}}"
  [^longs res]
  (let [ns      (aget res 6)
        shard   (fn [s] (vec (java.util.Arrays/copyOfRange res (int (+ 8 (* 10 s))) (int (+ 18 (* 10 s))))))
        eoff0   (+ 8 (* 10 ns))
        eoff    (fn [s] (aget res (int (+ eoff0 s))))
        elems0  (+ eoff0 ns 1)
        elem    (fn [e] (let [o (int (+ elems0 (* 4 e)))] [(aget res o) (aget res (+ o 1)) (aget res (+ o 2)) (aget res (+ o 3))]))
        n-elems (aget res 7)
        per     (vec
                 (for [s (range ns)]
                   (let [[valid attempt stable lost never stale dup] (shard s)
                         es      (map elem (range (eoff s) (eoff (inc s))))
                         by-out  (group-by second es)           ; 0 never-read, 1 stable, 2 lost
                         stale-e (->> (by-out 1) (filter #(pos? (nth % 2))) (sort-by #(- (nth % 2))))]
                     {:valid?            (verdict valid)
                      :attempt-count     attempt
                      :stable-count      stable
                      :lost-count        lost
                      :lost              (into (sorted-set) (map first (by-out 2)))
                      :never-read-count  never
                      :never-read        (into (sorted-set) (map first (by-out 0)))
                      :stale-count       stale
                      :stale             (into (sorted-set) (map first stale-e))
                      :worst-stale       (mapv (fn [[id _ lat]] {:element id :stable-latency lat}) (take 8 stale-e))
                      :stable-latencies  (quantiles (map #(nth % 2) (by-out 1)))
                      :lost-latencies    (quantiles (map #(nth % 2) (by-out 2)))
                      :duplicated-count  dup
                      :duplicated        (into (sorted-map) (keep (fn [[id _ _ d]] (when (> d 1) [id d])) es))})))
        sus0    (+ elems0 (* 4 n-elems))
        suspects (loop [k (int sus0) acc {}]
                   (if (>= k (alength res))
                     acc
                     (let [s (aget res k) idx (aget res (+ k 1)) nm (aget res (+ k 2))
                           miss (into (sorted-set) (java.util.Arrays/copyOfRange res (int (+ k 3)) (int (+ k 3 nm))))]
                       (recur (int (+ k 3 nm)) (update acc s (fnil conj []) [idx miss])))))]
    {:per-shard per :suspects suspects}))

(defn- check-set-full* [linearizable? history]
  (let [{:keys [arrays keys]} (flatten-history :set history)
        [h multi?] (handle)]
    (assoc (set-full-maps (Native/checkSetFull h multi? arrays (boolean linearizable?))) :keys keys)))

(defn set-full
  "Replacement for (checker/set-full {:linearizable? true}) — workloads/set_full.clj:157."
  [{:keys [linearizable?]}]
  (reify checker/Checker
    (check [_ _test history _opts]
      (first (:per-shard (check-set-full* linearizable? history))))))

(defn- raia-map [suspects]
  (if (seq suspects) {:valid? false :suspect-final-reads suspects} {:valid? true}))

(defn read-all-invoked-adds
  "Replacement for (read-all-invoked-adds) — workloads/set_full.clj:51-75; evaluated on the device in the same
  pass as set-full."
  []
  (reify checker/Checker
    (check [_ _test history _opts]
      (raia-map (get (:suspects (check-set-full* true history)) 0)))))

;; ---- bank -----------------------------------------------------------------------------------------------------
(defn bank-checker
  "Replacement for the ledger :SI checker — tests/ledger.clj:154-192 (same result map)."
  [{:keys [negative-balances?]}]
  (reify checker/Checker
    (check [_ test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :bank history)
            accts (set (:accounts test))
            total (long (:total-amount test 0))
            res   (Native/checkBankTotals @ctx arrays (int-array (:accounts test)) total (boolean negative-balances?))
            err   (fn [t idx]                          ; the error map check-op builds (tests/ledger.clj:127-152)
                    (let [op (first (filter #(= :read (:f %)) (keep ledger->bank-op [(by-index idx)])))
                          v  (:value op)]
                      (case (bank-error t)
                        :unexpected-key {:type :unexpected-key :unexpected (remove accts (clojure.core/keys v)) :op op}
                        :nil-balance    {:type :nil-balance :nils (into {} (remove val v)) :op op}
                        :wrong-total    {:type :wrong-total :total (reduce + (vals v)) :op op}
                        :negative-value {:type :negative-value :negative (filter neg? (vals v)) :op op})))
            at    (fn [base t] (aget res (int (+ base t))))     ; count 6.., first 11.., last 16.., worst 21..
            errors (into {}
                         (for [t [1 2 3 4] :when (pos? (at 6 t))]
                           [(bank-error t)
                            (merge {:count (at 6 t)
                                    :first (err t (at 11 t))
                                    :worst (err t (at 21 t))
                                    :last  (err t (at 16 t))}
                                   (when (= t 3)
                                     {:lowest (err t (aget res 28)) :highest (err t (aget res 29))}))]))
            out   {:valid?      (verdict (aget res 0))
                   :read-count  (aget res 2)
                   :error-count (aget res 3)
                   :first-error (when (pos? (aget res 3)) (err (aget res 5) (aget res 4)))
                   :errors      errors}]
        (if (pos? (aget res 1))
          ;; tests/ledger.clj:122-123: with :total-amount 0 err-badness divides by zero as soon as util/max-by
          ;; compares two :wrong-total errors -> the reference checker throws -> check-safe reports :unknown
          (assoc out :valid? :unknown
                 :error "java.lang.ArithmeticException: Divide by zero (err-badness, tests/ledger.clj:122-123)")
          out)))))

;; ---- monotonic keys -------------------------------------------------------------------------------------------
(def ^:private counter-field [:debits-posted :credits-posted])

(defn monotonic-key-checker
  "Elle's monotonic-key graph over the ledger's counters (src/tigerbeetle/elle/core.clj) plus real-time order, on the
  GPU: a cycle proves that no (real-time respecting) serial order explains the reads.  Add it to the compose map at
  tests/ledger.clj:363-367 as `:monotonic (monotonic-key-checker {})`; {:realtime? false} gives the literal
  elle/core.clj graph.  Result: {:valid? :read-count :key-count [:cause] [:op :cycle :steps]}."
  [{:keys [realtime?] :or {realtime? true}}]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-counters history)
            res  (Native/checkMonotonicKeys @ctx arrays (boolean realtime?))
            at   (fn [i] (aget res (int i)))
            s    6                                       ; shard 0: valid cause reads keys witness partner, edges
            step (fn [o] (if (= 1 (at o))
                           {:type :monotonic :key [(quot (at (+ o 1)) 2) (counter-field (rem (at (+ o 1)) 2))]
                            :value (at (+ o 2)) :value' (at (+ o 3))}
                           {:type :realtime :value (at (+ o 2)) :value' (at (+ o 3))}))]
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :key-count (at (+ s 3))}
          (= 1 (at s)) (assoc :cause (cause (at (+ s 1))))
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 4)))
                              :cycle [(by-index (at (+ s 5))) (by-index (at (+ s 4))) (by-index (at (+ s 5)))]
                              :steps [(step (+ s 6)) (step (+ s 10))]))))))

;; ---- counter bounds -------------------------------------------------------------------------------------------
(def ^:private cb-error-type {1 :below-completed-transfers 2 :above-invoked-transfers})

(defn counter-bounds-checker
  "Every counter an :ok ledger read observes against the transfers around it, on the GPU: at least the :ok transfers
  that completed before the read was invoked, at most the non-:fail transfers invoked before it completed.  Below is a
  lost transfer, above a phantom or duplicated one.  Add it to the compose map at tests/ledger.clj:363-367 as
  `:counter-bounds (counter-bounds-checker {})`.  Transfer txns with more than one [:t ...] micro-op throw (only the
  first is flattened, so the upper bounds would be too small), which check-safe reports as :unknown.
  Result: {:valid? :read-count :transfer-count :error-count [:op :error]}."
  [_opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [multi (count (filter (fn [{:keys [f type value]}]
                                   (and (= :txn f) (= :invoke type) (= :t (ffirst value)) (< 1 (count value))))
                                 history))
            _     (when (pos? multi)
                    (throw (IllegalArgumentException.
                             (str multi " transfer txns have more than one [:t ...] micro-op"))))
            {:keys [arrays by-index]} (flatten-history :ledger-counters history)
            res   (Native/checkCounterBounds @ctx arrays)
            at    (fn [i] (aget res (int i)))
            s     8                                      ; shard 0: valid reads transfers keys below above witness ...
            key   (at (+ s 7))]
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 1)) :transfer-count (at (+ s 2))
                 :error-count (+ (at (+ s 4)) (at (+ s 5)))}
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 6)))
                              :error {:type     (cb-error-type (at (+ s 8)))
                                      :key      [(quot key 2) (counter-field (rem key 2))]
                                      :value    (at (+ s 10))
                                      :bound    (at (+ s 11))
                                      :transfer (when (<= 0 (at (+ s 9))) (by-index (at (+ s 9))))}))))))

;; ---- transfer lookups ---------------------------------------------------------------------------------------
(def ^:private tl-kind {1 :phantom 2 :mismatch 3 :failed-visible 4 :future 5 :duplicate 6 :lost 7 :vanished
                        8 :read-below-lookup 9 :read-above-lookup})

(defn transfer-lookup-checker
  "The transfer records :ok [:l-t ...] lookups return, on the GPU, against the transfers clients issued (phantom,
  mismatched, failed, future and duplicate records), against each other and the :ok transfers (a transfer seen once
  must stay visible: lost, vanished), and against the counters reads show (read below / above a lookup's sums).
  :info transfers are never required to appear.  Add it to the compose map at tests/ledger.clj:363-367 as
  `:transfer-lookups (transfer-lookup-checker {})`.
  Result: {:valid? :lookup-count :record-count :transfer-count :read-count :error-count :errors [:op :error]}."
  [_opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res    (Native/checkTransferLookups @ctx arrays)
            at     (fn [i] (aget res (int i)))
            s      10                                     ; shard 0: valid lookups records transfers reads counts[9] ...
            errors (into {} (for [k (range 9) :let [n (at (+ s 5 k))] :when (pos? n)] [(tl-kind (inc k)) n]))
            kind   (at (+ s 15))
            key    (at (+ s 17))
            rel    (at (+ s 18))]
        (cond-> {:valid? (verdict (at s)) :lookup-count (at (+ s 1)) :record-count (at (+ s 2))
                 :transfer-count (at (+ s 3)) :read-count (at (+ s 4)) :error-count (reduce + (vals errors))
                 :errors errors}
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 14)))
                              :error (cond-> {:type (tl-kind kind)}
                                       (< kind 8)  (assoc :transfer-id (at (+ s 16)))
                                       (>= kind 8) (assoc :key   [(quot key 2) (counter-field (rem key 2))]
                                                          :value (at (+ s 19))
                                                          :bound (at (+ s 20)))
                                       (<= 0 rel)  (assoc :related (by-index rel)))))))))

;; ---- read explanations -------------------------------------------------------------------------------------
(def ^:private rx-kind {1 :key 2 :joint})

(defn read-explanation-checker
  "Whether one set of transfers explains every counter each :ok read shows, on the GPU: the transfers that must be in
  the read, the ones that cannot be and the ones that may be, and a budgeted search for a subset of the last that
  closes every counter at once.  :key errors have a counter no subset closes (lost, phantom, duplicated or corrupt
  amounts), :joint errors close each counter alone but not all at once (torn or fractured transfers).  A read the
  budget ({:max-nodes n}) does not decide makes the verdict :unknown.  Add it to the compose map at
  tests/ledger.clj:363-367 as `:read-explanations (read-explanation-checker {})`.
  Result: {:valid? :read-count :transfer-count :explained-count :undecided-count :error-count :errors [:op :error]}."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res    (Native/checkReadExplanations @ctx arrays (long (:max-nodes opts 0)))
            at     (fn [i] (aget res (int i)))
            s      11                                     ; shard 0: valid reads transfers witness explained undecided ...
            errors (into {} (for [k (range 2) :let [n (at (+ s 6 k))] :when (pos? n)] [(rx-kind (inc k)) n]))
            kind   (at (+ s 9))
            key    (at (+ s 10))]
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 1)) :transfer-count (at (+ s 2))
                 :explained-count (at (+ s 4)) :undecided-count (at (+ s 5)) :error-count (reduce + (vals errors))
                 :errors errors}
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 3)))
                              :error (cond-> {:type (rx-kind kind) :must-count (at (+ s 11)) :may-count (at (+ s 12))}
                                       (<= 0 key) (assoc :key [(quot key 2) (counter-field (rem key 2))])
                                       (= 1 kind) (assoc :value (at (+ s 13)) :must-sum (at (+ s 14))))))))))

;; ---- read gaps ----------------------------------------------------------------------------------------------------
(def ^:private rg-kind {1 :key 2 :joint 3 :double})

(defn read-gap-checker
  "Whether the transfers committed between two successive :ok reads explain what changed, on the GPU: the reads of a
  shard in the monotonic-key order (by the sum of their values, then invocation), and for each gap between neighbours a
  budgeted search for a subset of the transfers that may have committed inside it summing to the change of every
  counter.  :key errors have a counter that goes down or that no subset closes, :joint errors close each counter alone
  but not all at once, :double errors name a transfer two gaps both need.  A gap the budget ({:max-nodes n}) does not
  decide, and a shard with a partial read, make the verdict :unknown.  Add it to the compose map at
  tests/ledger.clj:363-367 as `:read-gaps (read-gap-checker {})`.
  Result: {:valid? :read-count :transfer-count :explained-count :undecided-count :error-count :errors
  [:op :lower-op :error]}."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res    (Native/checkReadGaps @ctx arrays (long (:max-nodes opts 0)))
            at     (fn [i] (aget res (int i)))
            s      12                                     ; shard 0: valid cause reads transfers explained undecided ...
            errors (into {} (for [k (range 3) :let [n (at (+ s 6 k))] :when (pos? n)] [(rg-kind (inc k)) n]))
            kind   (at (+ s 12))
            key    (at (+ s 13))]
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :explained-count (at (+ s 4)) :undecided-count (at (+ s 5)) :error-count (reduce + (vals errors))
                 :errors errors}
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 10)))
                              :error (cond-> {:type (rg-kind kind) :eligible-count (at (+ s 17))}
                                       (<= 0 key)  (assoc :key [(quot key 2) (counter-field (rem key 2))])
                                       (= 1 kind)  (assoc :delta (at (+ s 14)))
                                       (= 3 kind)  (assoc :transfer-id (at (+ s 15))
                                                          :other-op (by-index (at (+ s 16))))))
          (and (= 2 (at s)) (<= 0 (at (+ s 11)))) (assoc :lower-op (by-index (at (+ s 11)))))))))

;; ---- transfer placement -------------------------------------------------------------------------------------------
(def ^:private tp-kind {1 :key 2 :joint 3 :double 4 :lost})

(defn transfer-placement-checker
  "The read-gap check with located transfers carried across gaps, on the GPU: a transfer one gap's search proves it
  holds, or that only one gap of its window can still hold, is placed there and leaves the other gaps, which are
  searched again without it until nothing moves ({:max-rounds n}, default 64).  Besides the read-gap errors, :lost
  errors name a transfer known to be committed before some read that no gap can hold.  A gap the budget
  ({:max-nodes n}) does not decide, and a shard with a partial read, make the verdict :unknown.  Add it to the compose
  map at tests/ledger.clj:363-367 as `:transfer-placement (transfer-placement-checker {})`.
  Result: {:valid? :read-count :transfer-count :explained-count :undecided-count :error-count :errors :placed-count
  :rounds [:op :lower-op :error]}."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res    (Native/checkTransferPlacement @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0)))
            at     (fn [i] (aget res (int i)))
            s      15                                     ; shard 0: valid cause reads transfers explained undecided ...
            errors (into {} (for [k (range 4) :let [n (at (+ s 6 k))] :when (pos? n)] [(tp-kind (inc k)) n]))
            kind   (at (+ s 15))
            key    (at (+ s 16))]
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :explained-count (at (+ s 4)) :undecided-count (at (+ s 5)) :error-count (reduce + (vals errors))
                 :errors errors :placed-count (at (+ s 10)) :rounds (at (+ s 12))}
          (= 2 (at s)) (assoc :op    (by-index (at (+ s 13)))
                              :error (cond-> {:type (tp-kind kind) :round (at (+ s 17))
                                              :eligible-count (at (+ s 21))}
                                       (<= 0 key)       (assoc :key [(quot key 2) (counter-field (rem key 2))])
                                       (= 1 kind)       (assoc :delta (at (+ s 18)))
                                       (#{3 4} kind)    (assoc :transfer-id (at (+ s 19))
                                                               :other-op (by-index (at (+ s 20))))))
          (and (= 2 (at s)) (<= 0 (at (+ s 14)))) (assoc :lower-op (by-index (at (+ s 14)))))))))

(def ^:private sw-cause {4 :partial-read 5 :anomaly 6 :undecided 7 :no-witness 8 :real-time 9 :lookup})

(defn serial-witness-checker
  "A proof that a ledger history is linearizable, on the GPU, or :unknown: the transfer-placement check, then one
  explanation chosen per read gap (no transfer in two, {:max-rounds n} witness rounds) and the serial order they give
  checked against real time.  :valid? true means the reads and transfers are linearizable for the per-account
  counters, and so for the bank model with negative balances allowed (the :linear question); otherwise :unknown with a
  :cause (:partial-read, :anomaly, :undecided, :no-witness, :real-time), never false.  Add it to the compose map at
  tests/ledger.clj:363-367 as `:serial-witness (serial-witness-checker {})`.
  Result: {:valid? :read-count :transfer-count :committed-count :committed-crashed-count :after-count :rounds
  [:cause :op :transfer-id]}."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res (Native/checkSerialWitness @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0)))
            at  (fn [i] (aget res (int i)))
            s   12]                                        ; shard 0: valid cause reads transfers committed ...
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :committed-count (at (+ s 4)) :committed-crashed-count (at (+ s 5)) :after-count (at (+ s 6))
                 :rounds (at (+ s 8))}
          (pos? (at (+ s 1)))   (assoc :cause (sw-cause (at (+ s 1))))
          (<= 0 (at (+ s 9)))   (assoc :op (by-index (at (+ s 9))))
          (<= 0 (at (+ s 10)))  (assoc :transfer-id (at (+ s 10))))))))

(defn repaired-witness-checker
  "serial-witness-checker with repairs: a shard the serial witness leaves :no-witness or :real-time gets up to
  {:max-repairs n} repair rounds, each banning the (transfer, gap) pairs the failure blames and choosing the released
  gaps' explanations again.  :valid? true is the same proof; a history the serial witness proves comes back unchanged.
  Add it to the compose map at tests/ledger.clj:363-367 as `:repaired-witness (repaired-witness-checker {})`.
  Result: serial-witness-checker's map plus :repairs and :ban-count."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res (Native/checkRepairedWitness @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0))
                                             (int (:max-repairs opts 0)))
            at  (fn [i] (aget res (int i)))
            s   14]                                        ; shard 0: valid cause reads transfers committed ...
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :committed-count (at (+ s 4)) :committed-crashed-count (at (+ s 5)) :after-count (at (+ s 6))
                 :rounds (at (+ s 8)) :repairs (at (+ s 11)) :ban-count (at (+ s 12))}
          (pos? (at (+ s 1)))   (assoc :cause (sw-cause (at (+ s 1))))
          (<= 0 (at (+ s 9)))   (assoc :op (by-index (at (+ s 9))))
          (<= 0 (at (+ s 10)))  (assoc :transfer-id (at (+ s 10))))))))

(defn lifted-witness-checker
  "repaired-witness-checker with lifted bans: a shard whose repairs stop because a repair recorded no new ban gets up
  to {:max-lifts n} lift steps, each letting the failing gaps take back transfers their own bans held (once per pair)
  before the repairs resume.  :valid? true is the same proof; a history the repaired witness proves comes back
  unchanged.  Add it to the compose map at tests/ledger.clj:363-367 as `:lifted-witness (lifted-witness-checker {})`.
  Result: repaired-witness-checker's map plus :lifts and :lifted-count."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res (Native/checkLiftedWitness @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0))
                                           (int (:max-repairs opts 0)) (int (:max-lifts opts 0)))
            at  (fn [i] (aget res (int i)))
            s   16]                                        ; shard 0: valid cause reads transfers committed ...
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :committed-count (at (+ s 4)) :committed-crashed-count (at (+ s 5)) :after-count (at (+ s 6))
                 :rounds (at (+ s 8)) :repairs (at (+ s 11)) :ban-count (at (+ s 12)) :lifts (at (+ s 13))
                 :lifted-count (at (+ s 14))}
          (pos? (at (+ s 1)))   (assoc :cause (sw-cause (at (+ s 1))))
          (<= 0 (at (+ s 9)))   (assoc :op (by-index (at (+ s 9))))
          (<= 0 (at (+ s 10)))  (assoc :transfer-id (at (+ s 10))))))))

(defn class-witness-checker
  "lifted-witness-checker, then a class pass on every shard it leaves :unknown (undecided, no-witness or real-time):
  from the transfer-placement check's owners, witness rounds that treat crashed transfers with the same debit, credit,
  amount and lookup bounds as one class, gather at most as many of a class as a gap can use and hand each gap the
  earliest members.  :valid? true is the same proof; a history the lifted witness proves comes back unchanged.  Add it
  to the compose map at tests/ledger.clj:363-367 as `:class-witness (class-witness-checker {})`.  Result:
  lifted-witness-checker's map plus :class-rounds and :handed-count, and :class-cause when the class pass failed."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res (Native/checkClassWitness @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0))
                                          (int (:max-repairs opts 0)) (int (:max-lifts opts 0)))
            at  (fn [i] (aget res (int i)))
            s   18]                                        ; shard 0: valid cause reads transfers committed ...
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :committed-count (at (+ s 4)) :committed-crashed-count (at (+ s 5)) :after-count (at (+ s 6))
                 :rounds (at (+ s 8)) :repairs (at (+ s 11)) :ban-count (at (+ s 12)) :lifts (at (+ s 13))
                 :lifted-count (at (+ s 14)) :class-rounds (at (+ s 16)) :handed-count (at (+ s 17))}
          (pos? (at (+ s 1)))   (assoc :cause (sw-cause (at (+ s 1))))
          (pos? (at (+ s 15)))  (assoc :class-cause (sw-cause (at (+ s 15))))
          (<= 0 (at (+ s 9)))   (assoc :op (by-index (at (+ s 9))))
          (<= 0 (at (+ s 10)))  (assoc :transfer-id (at (+ s 10))))))))

(defn lookup-witness-checker
  "class-witness-checker, then every :ok lookup of a shard it proves placed in the serial order: each lookup where it
  returns exactly the transfers committed before it, the lookups of one read gap nested, and one real-time pass over
  the reads, transfers and lookups together.  :valid? true then covers the whole ledger history, lookups included.  A
  shard whose lookups have no place is :unknown with :cause :lookup and :lookup-op, the lookup that failed.  Add it to
  the compose map at tests/ledger.clj:363-367 as `:lookup-witness (lookup-witness-checker {})`.  Result:
  class-witness-checker's map plus :lookups-placed-count, and :lookup-cause and :lookup-op when the lookups failed."
  [opts]
  (reify checker/Checker
    (check [_ _test history _opts]
      (let [{:keys [arrays by-index]} (flatten-history :ledger-lookups history)
            res (Native/checkLookupWitness @ctx arrays (long (:max-nodes opts 0)) (int (:max-rounds opts 0))
                                           (int (:max-repairs opts 0)) (int (:max-lifts opts 0)))
            at  (fn [i] (aget res (int i)))
            s   19]                                        ; shard 0: valid cause reads transfers committed ...
        (cond-> {:valid? (verdict (at s)) :read-count (at (+ s 2)) :transfer-count (at (+ s 3))
                 :committed-count (at (+ s 4)) :committed-crashed-count (at (+ s 5)) :after-count (at (+ s 6))
                 :rounds (at (+ s 8)) :repairs (at (+ s 11)) :ban-count (at (+ s 12)) :lifts (at (+ s 13))
                 :lifted-count (at (+ s 14)) :class-rounds (at (+ s 16)) :handed-count (at (+ s 17))
                 :lookups-placed-count (at (+ s 20))}
          (pos? (at (+ s 1)))   (assoc :cause (sw-cause (at (+ s 1))))
          (pos? (at (+ s 15)))  (assoc :class-cause (sw-cause (at (+ s 15))))
          (pos? (at (+ s 18)))  (assoc :lookup-cause (sw-cause (at (+ s 18)))
                                       :lookup-op (by-index (at (+ s 19))))
          (<= 0 (at (+ s 9)))   (assoc :op (by-index (at (+ s 9))))
          (<= 0 (at (+ s 10)))  (assoc :transfer-id (at (+ s 10))))))))

;; ---- independent ----------------------------------------------------------------------------------------------
(defn independent-checker
  "Like (independent/checker (checker/compose checkers)) for a map {name checker-kind} built from THIS namespace's
  constructors, but ALL keys go to the native side in ONE call per checker kind — the GPU (or, with *n-gpus* > 1,
  the 8 GPUs of the box) owns the fan-out instead of a JVM thread pool.  Returns the same shape:
  {:valid? .. :results {k {name result .. :valid? ..}} :failures [k ..]}.
  `checkers` maps names to one of [:set-full opts] [:read-all-invoked-adds] [:linearizable opts]."
  [checkers]
  (reify checker/Checker
    (check [_ test history _opts]
      (let [sf   (delay (check-set-full* (boolean (some (fn [[_ [k o]]] (and (= k :set-full) (:linearizable? o))) checkers))
                                         history))
            cols (into {}
                       (for [[nm [kind o]] checkers]
                         [nm (case kind
                               :set-full              (zipmap (:keys @sf) (:per-shard @sf))
                               :read-all-invoked-adds (zipmap (:keys @sf)
                                                              (map-indexed (fn [s _] (raia-map (get (:suspects @sf) s)))
                                                                           (:keys @sf)))
                               :linearizable          (let [r (check-linearizable* (:model o) test history)]
                                                        (zipmap (:keys r) (:shards r))))]))
            ks      (sort (distinct (mapcat clojure.core/keys (vals cols))))
            results (into (sorted-map)
                          (for [k ks]
                            (let [m (into {} (for [[nm col] cols] [nm (get col k {:valid? :unknown})]))]
                              [k (assoc m :valid? (checker/merge-valid (map :valid? (vals m))))])))
            failures (vec (for [[k r] results :when (not (true? (:valid? r)))] k))]
        {:valid?   (checker/merge-valid (map :valid? (vals results)))
         :results  results
         :failures failures}))))
