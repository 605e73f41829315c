/*
 * rapid_b200 — C ABI of the H100-native cut-detection + fast-round-tally path of Rapid.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference (lalithsuresh/rapid) is Java; the classes
 * on the hot path — MembershipView, MultiNodeCutDetector, FastPaxos — are package-private concrete
 * classes constructed directly by Cluster.Builder / MembershipService, so the binding a maintainer adds is
 * a JNI veneer (java/com/vrg/rapid/gpu/Native.java + java/jni/rapid_jni.c, shown in INTEGRATION.md) whose
 * native methods are exactly the entry points below: plain pointers and sizes, no C++/torch types.
 *
 * Besides the path itself (view, cut detection, fast-round tally, sharded tally) the header carries the rows SURVEY.md §8f
 * marks "next": applying a decided cut, the classic-Paxos fallback (rapid_px_*, rapid_pxa_*), wire-format ingest
 * (rapid_wire_*) and alert generation by the edge failure detectors (rapid_fdet_*).
 *
 * Citations are relative to rapid/src/main/java/com/vrg/rapid/ in the reference repository.
 *
 * Conventions
 *   - every function returns an int32 status: RAPID_OK or a negative RAPID_E* code; rapid_last_error()
 *     gives the thread-local message.  No exception crosses the ABI.
 *   - handles are opaque, library-owned, freed by *_destroy; a handle is single-writer (the reference runs
 *     all protocol logic on one "protocol" thread, SharedResources.java:53); distinct handles may be used
 *     from distinct threads.
 *   - array arguments are caller-owned HOST memory unless the parameter name ends in _dev.
 *   - node ids: members are 0..n-1 in the order given to rapid_view_create; joiners registered with
 *     rapid_view_register_joiners get ids n, n+1, ...
 *   - the library needs a CUDA device: there is no CPU fallback; without one every create fails RAPID_ECUDA.
 */
#ifndef RAPID_B200_H
#define RAPID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built -fvisibility=hidden; only this header is exported */
#endif

#define RAPID_OK                0
#define RAPID_EINVAL           (-1)   /* bad K/H/L (MultiNodeCutDetector.java:52-55), ring >= K, bad size/id */
#define RAPID_ENOT_IN_RING     (-2)   /* MembershipView.NodeNotInRingException      (MembershipView.java:508-512) */
#define RAPID_EALREADY_IN_RING (-3)   /* MembershipView.NodeAlreadyInRingException  (:502-506) */
#define RAPID_EUUID_SEEN       (-4)   /* MembershipView.UUIDAlreadySeenException    (:514-519) */
#define RAPID_EHASH_COLLISION  (-5)   /* two endpoints tie on a ring key: the Java TreeSet would silently drop one */
#define RAPID_ECUDA            (-6)
#define RAPID_ENCCL            (-7)
#define RAPID_ENOMEM           (-8)
#define RAPID_EUNSUPPORTED     (-9)

#define RAPID_EDGE_UP   0   /* rapid.proto EdgeStatus */
#define RAPID_EDGE_DOWN 1

#define RAPID_MAX_K 14      /* ring-report bits 0..13 of the logical 16-bit per-(subject,receiver) state word (bucketed handles
                               store the ring bits only: 10 bits per receiver when K <= 10, 16 otherwise) */

typedef struct rapid_view rapid_view;   /* MembershipView: K rings in HBM (SoA)                       */
typedef struct rapid_cd   rapid_cd;     /* MultiNodeCutDetector state of R virtual nodes in HBM       */
typedef struct rapid_fp   rapid_fp;     /* FastPaxos fast-round tally of one configuration            */
typedef struct rapid_comm rapid_comm;   /* NCCL communicator for the sharded (multi-GPU) tally         */
typedef struct rapid_px   rapid_px;     /* classic-Paxos tallies of one node (coordinator + learner)   */
typedef struct rapid_pxa  rapid_pxa;    /* classic-Paxos acceptor state of R virtual nodes in HBM      */
typedef struct rapid_wire rapid_wire;   /* protobuf wire-format decoder bound to a view's dictionary    */
typedef struct rapid_fdet rapid_fdet;   /* the K edge failure detectors of every virtual node            */

const char* rapid_version(void);
int32_t rapid_last_error(char* buf, size_t cap);
int32_t rapid_device_count(int32_t* out);

/* ------------------------------------------------------------------------------------------------
 * MembershipView  (MembershipView.java)
 * ---------------------------------------------------------------------------------------------- */

/* Bulk constructor MembershipView(K, nodeIds, endpoints) (:74-89): ring k = endpoints ordered by the signed
 * 64-bit key  xx_k(hostname) * 31 + xx_k.hashInt(port)  (AddressComparator :562-587, XXH64 seed k).
 * host_bytes = hostnames concatenated, host_off[n+1] their offsets.  A key tie on any ring returns
 * RAPID_EALREADY_IN_RING if the two endpoints are identical, else RAPID_EHASH_COLLISION (we refuse rather than
 * silently drop like TreeSet.add).  n may be 0. */
int32_t rapid_view_create(rapid_view** out, int32_t K, int64_t n, const uint8_t* host_bytes,
                          const int32_t* host_off, const int32_t* port, int32_t device);
int32_t rapid_view_destroy(rapid_view* v);
int32_t rapid_view_size(const rapid_view* v, int64_t* out_n);                  /* getMembershipSize :425-432 */
int32_t rapid_view_ring(const rapid_view* v, int32_t k, int32_t* out_ids /*n*/);      /* getRing :380-388 */
int32_t rapid_view_keys(const rapid_view* v, int32_t k, int64_t* out_keys /*n, by node id*/);
/* getObserversOf :210-257 (ring successors) / getSubjectsOf :267-282 (ring predecessors).
 * *out_count = K, or 0 when the view has <= 1 member; RAPID_ENOT_IN_RING if node is not a member. */
int32_t rapid_view_observers(const rapid_view* v, int32_t node, int32_t* out /*K*/, int32_t* out_count);
int32_t rapid_view_subjects(const rapid_view* v, int32_t node, int32_t* out /*K*/, int32_t* out_count);
/* getExpectedObserversOf :292-303 — ring PREDECESSORS of where the endpoint would sit; works for non-members;
 * *out_count = 0 only for an empty view. */
int32_t rapid_view_expected_observers(const rapid_view* v, const uint8_t* host, int32_t len, int32_t port,
                                      int32_t* out /*K*/, int32_t* out_count);
/* getRingNumbers(observer, subject) :397-418 as a bitmask {k : subject is observer's predecessor on ring k}. */
int32_t rapid_view_ring_numbers(const rapid_view* v, int32_t observer, int32_t subject, uint16_t* out_mask);
/* All members at once: out_obs[i*K+k], out_subj[i*K+k] (-1 when the view has <= 1 member). */
int32_t rapid_view_tables(const rapid_view* v, int32_t* out_obs, int32_t* out_subj);
/* Configuration.getConfigurationId :544-556 over identifiersSeen (sorted by signed (high, low), :474-500)
 * followed by the ring-0 endpoint order. */
int32_t rapid_view_config_id(const rapid_view* v, const int64_t* id_high, const int64_t* id_low, int64_t n_ids,
                             int64_t* out);
/* Register joining endpoints (the edgeDst of UP alerts).  They get ids n.. ; their expected observers
 * (getExpectedObserversOf) and ring-0 keys are computed on device.  RAPID_EALREADY_IN_RING if one is a member. */
int32_t rapid_view_register_joiners(rapid_view* v, int64_t n_add, const uint8_t* host_bytes,
                                    const int32_t* host_off, const int32_t* port, int32_t* out_first_id);
int32_t rapid_view_num_joiners(const rapid_view* v, int64_t* out);
/* decideViewChange (MembershipService.java:385-444) on the view: every cut id that is a member is removed (ringDelete
 * :167-201), every other one must be a registered joiner and is added (ringAdd :123-160).  The K rings are UPDATED on the
 * device — order-preserving compaction of every ring + a sorted merge of the joiners, no re-hash or re-sort of the members;
 * the endpoint table, per-id keys and NodeIds are compacted alongside; only the cut ids (in) and status words (out) cross the
 * bus.  Ids are renumbered densely (surviving members in order, then the admitted joiners; joiners not in the cut are
 * dropped); out_old_to_new[n + joiners] receives the mapping (-1 = gone) and may be NULL.  With NodeIds set
 * (rapid_view_set_node_ids) an admitted joiner whose NodeId is already in identifiersSeen -> RAPID_EUUID_SEEN
 * (UUIDAlreadySeenException, MembershipView.java:126-128) and NOTHING changes.  A cut that admits one endpoint twice (registered
 * twice as a joiner) -> RAPID_EALREADY_IN_RING (the second ringAdd's NodeAlreadyInRingException); two different endpoints with
 * equal keys on a ring -> RAPID_EHASH_COLLISION.  Every refusal leaves the view, identifiersSeen included, as it was, and
 * out_old_to_new unwritten.  Detector handles created on the old view must be
 * destroyed and recreated (their receivers are ring-0 positions of that view). */
int32_t rapid_view_apply_cut(rapid_view* v, const int32_t* cut_ids, int64_t n_cut, int32_t* out_old_to_new);
/* identifiersSeen on the device (MembershipView.java:58-60): NodeIds of the current members (index = node id) seed it —
 * RAPID_EUUID_SEEN if two members share one; the NodeIds of registered joiners [first_joiner_id, +count) come from their UP
 * alerts (MembershipService.java:677-685) and join the set when a cut admits them; ids of removed nodes stay (:167-201).
 * rapid_view_current_config_id = getCurrentConfigurationId (:360-372, :544-556) from that set and ring 0: 8 bytes leave the device. */
int32_t rapid_view_set_node_ids(rapid_view* v, const int64_t* id_high, const int64_t* id_low);
int32_t rapid_view_set_joiner_ids(rapid_view* v, int32_t first_joiner_id, int64_t count, const int64_t* id_high, const int64_t* id_low);
int32_t rapid_view_current_config_id(const rapid_view* v, int64_t* out);
/* expected observers of every registered joiner: out[j*K+k] for joiner id n + j. */
int32_t rapid_view_joiner_tables(const rapid_view* v, int32_t* out);
/* Expansion of the monitoring overlay.  The observer graph of the view's n >= 3 members is A = sum_k (P_k + P_k^T), P_k the
 * permutation "successor on ring k": A[v][obs[v][k]] += 1 and A[v][subj[v][k]] += 1 for every k, multiplicities kept (a node that
 * observes another on m rings contributes m).  A is symmetric, its rows sum to 2K, its top eigenvalue is 2K with the all-ones
 * vector.  For A restricted to the complement of that vector: *lambda2 = the largest eigenvalue, *lambda_min = the smallest;
 * max(|lambda2|, |lambda_min|) / 2K is the expander figure of the Rapid paper (< 0.45 at K = 10).  Registered joiners are not part
 * of the graph.  Computed on the device by Lanczos with full re-orthogonalisation in fp64 (basis in HBM: steps * n * 8 bytes of
 * scratch for the duration of the call), from the start vector  x[v] = 2 u - 1, u = (splitmix64(seed + v) >> 11) * 2^-53,  mean
 * removed, normalised.  It stops when *residual <= tol * 2K or after max_steps operator applications (or n - 1, the dimension of
 * the complement), whichever comes first; reaching max_steps is not an error.  *residual = the larger |beta_m * s_m| of the two
 * reported Ritz values: each lies within it of an eigenvalue of A.  *steps = operator applications spent, *device_ms = CUDA events
 * around them.  Every out pointer may be NULL.  The same seed on the same view returns the same bits.  The view is not modified.
 * RAPID_EINVAL, and nothing is written, if n < 3 (n = 2 is bipartite with +-2K, n = 1 has no complement), tol <= 0 or max_steps
 * outside [2, RAPID_OVERLAY_MAX_STEPS]. */
#define RAPID_OVERLAY_MAX_STEPS 512
int32_t rapid_view_overlay_spectrum(const rapid_view* v, uint64_t seed, double tol, int32_t max_steps, double* lambda2,
                                    double* lambda_min, double* residual, int32_t* steps, float* device_ms);

/* ------------------------------------------------------------------------------------------------
 * MultiNodeCutDetector for R virtual nodes ("receivers")   (MultiNodeCutDetector.java,
 * MembershipService.java:300-354 batch driver, :644-675 filter)
 *
 * Receiver r (0 <= r < n_receivers) is the virtual node at ring-0 position receiver_begin + r, i.e. a shard
 * is a contiguous range of the ring-0 hash order.  State per (subject slot, receiver) is one uint16 in HBM,
 * laid out [slot][receiver] so that a warp touches consecutive receivers.
 * ---------------------------------------------------------------------------------------------- */

/* mode flags for rapid_cd_create */
#define RAPID_CD_SERVICE   0u   /* MembershipService semantics: filter, announcedProposal gating, union per batch */
#define RAPID_CD_RAW       1u   /* bare MultiNodeCutDetector semantics (aggregate / invalidate calls)             */
#define RAPID_CD_SWEEP     2u   /* force the per-cell sweep kernel (exact counters; the simple path)               */
#define RAPID_CD_BUCKETED  4u   /* force the subject-bucketed kernels (the fast path; SERVICE mode only)            */
#define RAPID_CD_LOG       8u   /* bucketed handles: keep the epoch's filtered cells (6 B per cell + the blocked flags) so
                                 * that rapid_cd_num_proposals can replay one receiver exactly; cleared by rapid_cd_clear  */

/* delivery description: which receiver gets which cells, in which order */
#define RAPID_DELIVERY_BLOCKED  1u   /* blocked[r] != 0: receiver r receives nothing this batch             */
#define RAPID_DELIVERY_BITMAP   2u   /* bitmap[cell][ceil(R/32)]: bit (r&31) of word r>>5 set = delivered   */
#define RAPID_DELIVERY_PERMUTED 4u   /* receiver r applies its cells in ascending
                                        splitmix64( splitmix64(perm_seed + receiver_begin + r) ^ cell_index ) */
#define RAPID_DELIVERY_SHUFFLED_BATCHES 8u
/* RAPID_DELIVERY_SHUFFLED_BATCHES — rapid_cd_apply_batches / rapid_cd_apply_batches_dev on SERVICE sweep handles (RAPID_CD_SWEEP)
 * only, alone or with BLOCKED: every receiver meets the n batches of the sequence in its own pseudo-random order, as the
 * reference's per-sender shuffled recipient lists make it (UnicastToAllBroadcaster.java:59-62), and the cells of each batch in
 * array order.  Receiver r (global index g = receiver_begin + r) handles batch P_g(j) at its step j = 0..n-1:
 *     if n <= 1: identity
 *     w   = smallest integer >= 4 with 4^w >= n;   m = 2^w - 1     (w >= 4: narrower halves skew the orders of small n)
 *     key = splitmix64(perm_seed + g)
 *     f(i, x) = splitmix64(key ^ ((uint64)(i + 1) << 58) ^ x) & m          for rounds i = 0..3
 *     E(v): a = v >> w; b = v & m; 4 times: (a, b) = (b, a ^ f(i, b)); return (a << w) | b
 *     P_g(j): v = E(j); while v >= n: v = E(v); return v                  (a bijection of [0, n))
 * announced_in[r] is the array index of the announcing batch.  Bucketed and RAW handles refuse it (RAPID_EUNSUPPORTED); with
 * PERMUTED or BITMAP, or on a single-batch entry point, it is RAPID_EINVAL.  A refused call changes nothing. */
typedef struct rapid_delivery {
    uint32_t        flags;
    const uint8_t*  blocked;     /* [R]                    (host) */
    const uint32_t* bitmap;      /* [n_cells][ceil(R/32)]  (host) */
    uint64_t        perm_seed;
} rapid_delivery;

/* ctor validation of MultiNodeCutDetector.java:51-55 (H <= K, L <= H, K >= 3, L > 0) -> RAPID_EINVAL.
 * K comes from the view.  max_subjects bounds the number of distinct subjects per configuration epoch
 * (0 = default). */
int32_t rapid_cd_create(rapid_cd** out, const rapid_view* v, int32_t H, int32_t L, int64_t n_receivers,
                        int64_t receiver_begin, uint32_t mode_flags, int64_t max_subjects);
int32_t rapid_cd_destroy(rapid_cd* cd);

/* One BatchedAlertMessage worth of alert cells applied to every receiver:  filter (cfg match, UP => dst not a
 * member, DOWN => dst a member; MembershipService.java:644-675)  ->  aggregateForProposal per cell in order
 * (MultiNodeCutDetector.java:84-128)  ->  invalidateFailingEdges (:137-164)  ->  union  ->  announcedProposal
 * (MembershipService.java:318-348).  A cell is one (edgeSrc, edgeDst, ring, status) report; an AlertMessage with r
 * ring numbers is r consecutive cells.  cell_cfg == NULL means every cell carries cfg_id.  delivery == NULL
 * means every receiver gets every cell in array order.
 * A cell whose ring number is >= K or whose edgeDst is not a known id is DROPPED, the rest of the batch is applied, and the
 * call returns RAPID_EINVAL naming the cell (the Java trusts ring numbers: only an `assert`, MultiNodeCutDetector.java:87).
 * Outputs (each may be NULL), per receiver:
 *   proposal_hash / proposal_hash2 : order-independent 128-bit fingerprint of the proposal announced by THIS batch
 *                                    (see rapid_proposal_fingerprint), 0 if none
 *   proposal_len                   : its size (0 if none)
 *   announced                      : announcedProposal after the batch */
int32_t rapid_cd_apply_batch(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src, const int32_t* dst,
                             const uint8_t* ring, const uint8_t* status, const int64_t* cell_cfg,
                             const rapid_delivery* delivery, uint64_t* proposal_hash, uint64_t* proposal_hash2,
                             int32_t* proposal_len, uint8_t* announced);
/* A SEQUENCE of BatchedAlertMessages in one call — one per sender, as the reference's AlertBatcher produces them
 * (MembershipService.java:613-637): batch b = cells [batch_off[b], batch_off[b+1]), batch_off[0] = 0, batch_off[n_batches] = n_cells.
 * Every receiver runs handleMessage (:300-354) once per batch, in array order: filter, cells, invalidateFailingEdges, and the
 * announcedProposal gating BETWEEN batches — a receiver that announces in batch b ignores batches b+1.. (:318-319).  Outputs as
 * rapid_cd_apply_batch (the proposal is that of the announcing batch), plus announced_in[receiver] = index of the batch in
 * which it announced during this call (-1: it did not).
 * Sweep handles walk the cells per receiver; delivery may carry BLOCKED / BITMAP.
 * Subject-bucketed handles (the default) first treat the whole sequence in ONE pass over the detector state — every batch
 * before the last folded, order-independently, into the state the last batch is applied to — which is exact whenever no
 * receiver emits a proposal before the last batch and no invalidation pass at the end of an earlier batch adds a report; both
 * premises are checked per receiver on the device before anything is committed, and if one fails for any receiver the
 * sequence is replayed batch by batch (always exact; rapid_cd_sequence_stats counts both outcomes).  delivery may carry
 * BLOCKED, PERMUTED (batch b is delivered to receiver r in the order of perm_seed + b) or BITMAP (always batch by batch). */
int32_t rapid_cd_apply_batches(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src, const int32_t* dst,
                               const uint8_t* ring, const uint8_t* status, const int64_t* cell_cfg, int64_t n_batches,
                               const int64_t* batch_off, const rapid_delivery* delivery, uint64_t* proposal_hash,
                               uint64_t* proposal_hash2, int32_t* proposal_len, uint8_t* announced, int32_t* announced_in);
/* rapid_cd_apply_batches with the cell arrays (and delivery arrays) already resident in device memory; batch_off stays a HOST
 * array.  Results stay on the device: rapid_fp_tally_cd counts every receiver that announced during the call,
 * rapid_cd_read_outputs / rapid_cd_read_announced_in copy them out. */
int32_t rapid_cd_apply_batches_dev(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev, const int32_t* dst_dev,
                                   const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev,
                                   int64_t n_batches, const int64_t* batch_off, const rapid_delivery* delivery_dev);
int32_t rapid_cd_read_announced_in(const rapid_cd* cd, int32_t* announced_in /* [R] */);
/* How many sequences this handle served in one pass / had to replay batch by batch, and — for the last refused attempt — how many
 * receivers failed either premise (a proposal could have been emitted before the last batch / an implicit report would have been
 * added at the end of an earlier batch).  Diagnostics; any pointer may be NULL. */
int32_t rapid_cd_sequence_stats(const rapid_cd* cd, int32_t* one_pass, int32_t* replayed, int32_t* refused_a1, int32_t* refused_a2);
/* Same as rapid_cd_apply_batch, with the cell arrays (and delivery arrays) already resident in device memory and no per-receiver
 * readback: results stay on the device for rapid_fp_tally_cd / rapid_cd_read_outputs. */
int32_t rapid_cd_apply_batch_dev(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev,
                                 const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                                 const int64_t* cell_cfg_dev, const rapid_delivery* delivery_dev);
/* Same as rapid_cd_apply_batch_dev, but only ENQUEUES the batch on the handle's stream and returns ("calls are synchronous
 * unless *_async", SURVEY.md §8b): a batch is three kernel launches with no host round trip in between, and rapid_fp_tally_cd
 * orders itself after it on the device, so a whole step (batch -> proposals -> votes -> decision) costs ONE host
 * synchronisation — the tally's read-back.  Subject-bucketed handles only.  The batch's status is collected at the next
 * synchronisation point (rapid_cd_sync, rapid_fp_tally_cd, or any accessor): dropped cells -> RAPID_EINVAL; a batch that needed
 * more than max_subjects subject slots is NOT applied -> RAPID_ENOMEM (the synchronous entry points grow the handle and replay
 * instead).  The device arrays must stay valid until then. */
int32_t rapid_cd_apply_batch_dev_async(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev,
                                       const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                                       const int64_t* cell_cfg_dev, const rapid_delivery* delivery_dev);
/* Wait for everything enqueued on the handle; returns (and clears) the latched status of asynchronous batches. */
int32_t rapid_cd_sync(rapid_cd* cd);
int32_t rapid_cd_read_outputs(const rapid_cd* cd, uint64_t* proposal_hash, uint64_t* proposal_hash2,
                              int32_t* proposal_len, uint8_t* announced);
/* The proposal receiver r announced, in canonical order = sorted by the ring-0 comparator
 * (MembershipService.java:346-348). */
int32_t rapid_cd_get_proposal(const rapid_cd* cd, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len);
/* Census of the receivers that announced in cd's last call (those rapid_fp_tally_cd counts): *n_classes distinct proposals,
 * *n_entries ids over all their lists.  Class c is the c-th lowest receiver of a distinct (hash, hash2, len) in receiver order (the
 * wire encoder's body numbering); its list is rapid_cd_get_proposal(its representative), each entry with a status,
 * RAPID_EDGE_DOWN for a member and RAPID_EDGE_UP for a registered joiner (VIEW_CHANGE_PROPOSAL's NodeStatusChange list,
 * MembershipService.java:336-345, :586-593).  cut_ids may be NULL (then in_cut reads -1); else in_cut[c] = entries of class c in
 * the cut.  Results stay on the handle until the next census; a refused call leaves the previous census bit-identical.
 * RAPID_EINVAL: a RAW handle, a handle that has applied no batch or was created before the view's members last changed, cut ids
 * outside [0, members + registered joiners) or repeated.  On a sharded handle representatives are local receiver indices.
 * Waits for the handle's asynchronous batches; synchronises once, for the counts. */
int32_t rapid_cd_proposal_census(rapid_cd* cd, const int32_t* cut_ids, int32_t cut_len, int64_t* n_classes, int64_t* n_entries);
/* any pointer may be NULL; arrays sized by the counts above (list_off: n_classes + 1; class c's entries are
 * ids[list_off[c] .. list_off[c + 1])) */
int32_t rapid_cd_read_census(const rapid_cd* cd, uint64_t* hash, uint64_t* hash2, int32_t* len, int32_t* voters,
                             int32_t* representative, int32_t* in_cut, int64_t* list_off, int32_t* ids, uint8_t* status);
/* class of every receiver, [R], -1 = did not announce: device memory of the handle, valid until the next census */
int32_t rapid_cd_census_classes_dev(const rapid_cd* cd, const int32_t** cls_dev);
int32_t rapid_cd_read_census_classes(const rapid_cd* cd, int32_t* cls);
/* getNumProposals :62-66 (the reference's tests are its only caller).  Sweep handles count while they walk the cells.
 * Subject-bucketed handles never see a receiver's cells in order, so they answer by REPLAYING that one receiver's cells from the
 * epoch's cell log, in its own order, through the sweep kernel — exact; needs RAPID_CD_LOG at creation (RAPID_EUNSUPPORTED
 * otherwise, or once the epoch held a per-receiver BITMAP delivery or more than 2^24 cells). */
int32_t rapid_cd_num_proposals(const rapid_cd* cd, int64_t receiver, int32_t* out);
/* clear() :169-178 + announcedProposal = false (MembershipService.java:425-426) for every receiver. */
int32_t rapid_cd_clear(rapid_cd* cd);
/* Parity aid: the ring-report bitmask per subject for one receiver (reportsPerHost as bitmasks). */
int32_t rapid_cd_debug_masks(const rapid_cd* cd, int64_t receiver, int32_t* out_subject_ids, uint16_t* out_masks,
                             int32_t cap, int32_t* out_n);
int32_t rapid_cd_debug_counters(const rapid_cd* cd, int64_t receiver, int32_t* updates_in_progress,
                                int32_t* seen_link_down);
/* Which kernel family served the last batch: 1 = sweep, 2 = bucketed-uniform, 3 = bucketed-generic (per-receiver delivery
 * bitmaps), 4 = bucketed-permuted (every cell to every receiver in its own order: the uniform kernel, moments on demand);
 * *n_kernel_launches = CUDA kernels launched by the last apply call. */
int32_t rapid_cd_last_path(const rapid_cd* cd, int32_t* path, int32_t* n_kernel_launches);
/* Bucketed handles, last batch: receivers that needed the exact interval analysis, (tile, subject) pairs on the
 * invalidation work list, distinct subjects and valid cells of the batch. */
int32_t rapid_cd_debug_stats(const rapid_cd* cd, int32_t* n_mixed, int32_t* n_inval_pairs, int32_t* n_batch_subjects,
                             int32_t* n_valid_cells);
/* Bucketed handles, last batch: the subject chunks of the apply kernel's grid (RAPID_B200_CHUNKS overrides the host's choice)
 * and the blocks of k_prepare's cooperative grid (RAPID_B200_PREP_GRID).  A sweep handle reports 0 chunks. */
int32_t rapid_cd_debug_grid(const rapid_cd* cd, int32_t* apply_chunks, int32_t* prepare_blocks);

/* RAW mode (RAPID_CD_RAW handles): the bare detector API the reference's CutDetectionTest drives.
 * aggregateForProposal(AlertMessage) :76-82 for every receiver (no filter, no announced gating); returns the
 * endpoints emitted for `receiver` by this call. */
int32_t rapid_cd_aggregate(rapid_cd* cd, int64_t n_cells, const int32_t* src, const int32_t* dst,
                           const uint8_t* ring, const uint8_t* status, int64_t receiver, int32_t* out_ids,
                           int32_t cap, int32_t* out_len);
/* invalidateFailingEdges(view) :137-164 */
int32_t rapid_cd_invalidate(rapid_cd* cd, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len);

/* Fingerprint of a proposal (a SET of node ids): h1 = sum mix1(id), h2 = sum mix2(id) (mod 2^64). */
int32_t rapid_proposal_fingerprint(const int32_t* ids, int64_t n, uint64_t* h1, uint64_t* h2);

/* ------------------------------------------------------------------------------------------------
 * FastPaxos fast round  (FastPaxos.java:125-156 handleFastRoundProposal)
 * ---------------------------------------------------------------------------------------------- */
/* One instance per configuration (FastPaxos ctor :61-85).  sender ids are int32 in [0, sender_capacity);
 * senders need not be members (the reference never checks). */
int32_t rapid_fp_create(rapid_fp** out, int64_t cfg_id, int64_t membership_size, int64_t sender_capacity,
                        int32_t device);
int32_t rapid_fp_destroy(rapid_fp* fp);
/* Start over for the next configuration (the new FastPaxos of MembershipService.java:427-429) on the same buffers. */
int32_t rapid_fp_reset(rapid_fp* fp, int64_t cfg_id, int64_t membership_size);
/* Apply n_votes FastRoundPhase2bMessages in array order: ignore if vote_cfg != cfg (:126), sender already
 * voted (:134) or already decided (:138); count identical proposals; decide when count >= N - floor((N-1)/4)
 * (:145-150).  A proposal is identified by (hash, hash2, len) = rapid_proposal_fingerprint + size.
 * vote_cfg / proposal_hash2 / proposal_len may be NULL (= cfg / 0 / 0).
 * Outputs: decided, the decided fingerprint, its vote count at the moment of decision (== quorum) and
 * votesReceived.size() at that moment (or the running totals if undecided).
 * A call is refused as a whole, and changes nothing, if a sender lies outside [0, sender_capacity) (RAPID_EINVAL) or if
 * more than 8 proposals reach the quorum within it (RAPID_EUNSUPPORTED).  Once decided, a call returns the decision
 * without looking at its votes. */
int32_t rapid_fp_tally(rapid_fp* fp, int64_t n_votes, const int32_t* sender, const int64_t* vote_cfg,
                       const uint64_t* proposal_hash, const uint64_t* proposal_hash2, const int32_t* proposal_len,
                       int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len,
                       int32_t* decided_count, int32_t* votes_received);
/* Votes straight from the detector's device-resident outputs: every receiver that announced a proposal in the last
 * batch votes for it (FastPaxos.propose :94-108; sender = its node id).  comm == NULL: single GPU.  comm != NULL:
 * every rank calls this with its shard; the local proposal-hash histograms are combined with one NCCL
 * all-reduce (plus a small verification all-reduce) and every rank gets the same answer. */
int32_t rapid_fp_tally_cd(rapid_fp* fp, const rapid_cd* cd, rapid_comm* comm, int32_t* decided,
                          uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len,
                          int32_t* decided_count, int32_t* votes_received);
/* The same in two halves: rapid_fp_tally_cd_async only ENQUEUES the tally (ordered on the device after whatever is in flight on
 * the detector, asynchronous batches included); rapid_fp_result waits for the LAST enqueued tally and reads the outcome.  A
 * whole stream of batches can thus be applied and tallied with one host synchronisation at the end: once a proposal has reached
 * the quorum later votes are ignored on the device (:138) and the decision is kept.  *decided_in_call = index (since
 * rapid_fp_reset) of the tally call that decided, -1 if undecided. */
int32_t rapid_fp_tally_cd_async(rapid_fp* fp, const rapid_cd* cd, rapid_comm* comm);
/* One configuration epoch of a virtual cluster enqueued in ONE call: rapid_cd_clear + rapid_fp_reset (decideViewChange's resets,
 * MembershipService.java:425-429) + rapid_cd_apply_batch_dev_async + rapid_fp_tally_cd_async.  Collect with rapid_fp_result. */
int32_t rapid_fp_epoch_async(rapid_fp* fp, rapid_cd* cd, rapid_comm* comm, int64_t cfg_id, int64_t membership_size, int64_t n_cells,
                             const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev,
                             const rapid_delivery* delivery_dev);
int32_t rapid_fp_result(rapid_fp* fp, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len,
                        int32_t* decided_count, int32_t* votes_received, int32_t* decided_in_call);
int32_t rapid_fp_quorum(int64_t membership_size, int64_t* out);   /* N - floor((N-1)/4) */
/* Device-side stopwatch over a whole sequence of (asynchronous) calls on a detector and its tally: rapid_cd_timer_start records a
 * CUDA event on the detector's stream, rapid_fp_timer_stop one on the tally's stream after everything enqueued so far on both,
 * waits for it and returns the milliseconds in between — kernels, copies AND the idle gaps between them. */
int32_t rapid_cd_timer_start(rapid_cd* cd);
int32_t rapid_fp_timer_stop(rapid_fp* fp, const rapid_cd* cd, float* out_ms);

/* ------------------------------------------------------------------------------------------------
 * Classic-Paxos fallback  (Paxos.java; SURVEY.md §8 f2)
 * A value (List<Endpoint>) is identified by an opaque (hash, hash2, len) triple the caller chooses (for the canonical
 * fast-round proposals: rapid_proposal_fingerprint + size); len == 0 is the empty list.  A Rank (rapid.proto:133-137)
 * is the pair (round, node_index), ordered by signed round then signed node_index (compareRanks :333-339).
 * All arrays are host memory, one element per message, in ARRIVAL order.
 * ---------------------------------------------------------------------------------------------- */
/* One node's tallies (Paxos ctor :76-90): the coordinator's Phase1b list and the learner's Phase2b sets, on the device.
 * message_capacity sizes the Phase1b list (it grows if exceeded) and bounds the distinct (rnd, sender) Phase2b pairs plus
 * rounds (RAPID_ENOMEM beyond ~3x message_capacity entries). */
int32_t rapid_px_create(rapid_px** out, int64_t cfg_id, int64_t membership_size, int64_t message_capacity, int32_t device);
int32_t rapid_px_destroy(rapid_px* px);
/* Start over for the next configuration (the new Paxos of FastPaxos.java:86 / MembershipService.java:427-429). */
int32_t rapid_px_reset(rapid_px* px, int64_t cfg_id, int64_t membership_size);
/* startPhase1a :98-113: *started = 0 if crnd.round > round, else crnd = (round, node_index) and *started = 1.
 * node_index stands for myAddr.hashCode() (:102). */
int32_t rapid_px_start_phase1a(rapid_px* px, int32_t round, int32_t node_index, int32_t* started);
/* selectProposalUsingCoordinatorRule :271-328 over n Phase1bMessages (stateless; N = the handle's membership size):
 * *chosen_index = index of the message whose vval is the chosen value, -1 if the chosen value is the empty list.
 * n == 0 is RAPID_EINVAL (the reference throws IllegalArgumentException :274). */
int32_t rapid_px_coordinator_rule(rapid_px* px, int64_t n, const int32_t* vrnd_round, const int32_t* vrnd_node,
                                  const uint64_t* vval_hash, const uint64_t* vval_hash2, const int32_t* vval_len,
                                  int64_t* chosen_index);
/* handlePhase1bMessage :159-191 for n messages: ignore if msg_cfg != cfg (:160) or rnd != crnd (:165); append; once more
 * than N/2 messages are held, the coordinator rule runs at every arrival and the first non-empty result becomes cval
 * (a Phase2aMessage{rnd = crnd, vval = cval} is broadcast, once).  msg_cfg / vval_hash2 may be NULL (= cfg / 0).
 * Outputs: *proposed = 1 iff THIS call picked cval; then *trigger_index = index (in this call's arrays) of the message at
 * which it happened and cval_* = the value.  *n_messages = phase1bMessages.size() after the call. */
int32_t rapid_px_phase1b(rapid_px* px, int64_t n, const int64_t* msg_cfg, const int32_t* rnd_round, const int32_t* rnd_node,
                         const int32_t* vrnd_round, const int32_t* vrnd_node, const uint64_t* vval_hash,
                         const uint64_t* vval_hash2, const int32_t* vval_len, int32_t* proposed, int64_t* trigger_index,
                         uint64_t* cval_hash, uint64_t* cval_hash2, int32_t* cval_len, int64_t* n_messages);
/* handlePhase2bMessage :223-236 for n messages: ignore if msg_cfg != cfg; acceptResponses[rnd].put(sender, msg); the
 * node decides at the first arrival that leaves more than N/2 distinct senders in that message's round, on THAT message's
 * value (:231-235).  Outputs: *decided = 1 iff the node has decided (now or earlier); if THIS call decided,
 * *decided_index = index of the deciding message (else -1); decided_* = the decision. */
int32_t rapid_px_phase2b(rapid_px* px, int64_t n, const int64_t* msg_cfg, const int32_t* rnd_round, const int32_t* rnd_node,
                         const int32_t* sender, const uint64_t* hash, const uint64_t* hash2, const int32_t* len,
                         int32_t* decided, int64_t* decided_index, uint64_t* decided_hash, uint64_t* decided_hash2,
                         int32_t* decided_len);
int32_t rapid_px_last_device_ms(const rapid_px* px, float* total_ms);

/* Acceptor state (rnd, vrnd, vval :63-65) of n_acceptors virtual nodes, resident in HBM; acceptor r is node
 * acceptor_begin + r (its `sender` id in the messages it emits). */
int32_t rapid_pxa_create(rapid_pxa** out, int64_t cfg_id, int64_t n_acceptors, int64_t acceptor_begin, int32_t device);
int32_t rapid_pxa_destroy(rapid_pxa* a);
int32_t rapid_pxa_reset(rapid_pxa* a, int64_t cfg_id);      /* rnd = vrnd = (0, 0), vval = [] (:82-85) for every acceptor */
/* registerFastRoundVote :244-257 for the listed acceptors (local indexes): skipped where rnd.round > 1, else
 * rnd = vrnd = (1, 1), vval = the vote.  An acceptor listed more than once ends with its LAST listed vote, whole, as calls
 * made one by one in list order would leave it.  An index outside [0, n_acceptors) gives RAPID_EINVAL and changes no
 * acceptor.  n <= 0x7ffffff0. */
int32_t rapid_pxa_register_fast_round_votes(rapid_pxa* a, int64_t n, const int64_t* acceptor, const uint64_t* hash,
                                            const uint64_t* hash2, const int32_t* len);
/* Same, straight from a detector's device-resident outputs: every receiver that announced a proposal in the last batch
 * registers it (FastPaxos.propose :94-98).  The detector's receivers must be this handle's acceptors (same count). */
int32_t rapid_pxa_register_fast_round_votes_cd(rapid_pxa* a, const rapid_cd* cd);
/* handlePhase1aMessage :120-151 of every acceptor for ONE broadcast Phase1aMessage: acceptors with rnd < rank adopt it
 * and answer Phase1bMessage{rnd = rank, vrnd, vval}.  The answers stay on the device; *n_replies = how many. */
int32_t rapid_pxa_phase1a(rapid_pxa* a, int64_t msg_cfg, int32_t round, int32_t node_index, int64_t* n_replies);
/* handlePhase2aMessage :198-216 of every acceptor for ONE broadcast Phase2aMessage: acceptors with rnd <= msg.rnd and
 * vrnd != msg.rnd accept (rnd = vrnd = msg.rnd, vval = msg.vval) and broadcast Phase2bMessage.  *n_accepted = how many. */
int32_t rapid_pxa_phase2a(rapid_pxa* a, int64_t msg_cfg, int32_t round, int32_t node_index, uint64_t hash, uint64_t hash2,
                          int32_t len, int64_t* n_accepted);
/* Deliver the device-resident answers of the last rapid_pxa_phase1a / rapid_pxa_phase2a to a coordinator / learner: the
 * answers of the n_shards acceptor handles listed (1..64 per rank, any order) and, with comm != NULL, of every other rank's
 * shards, delivered as one handle holding the union of their acceptors would: in ascending sender (perm_seed == 0) or in
 * ascending splitmix64(perm_seed ^ sender) order.  Outputs as in rapid_px_phase1b / rapid_px_phase2b; trigger_index /
 * decided_index are positions in that arrival order.  One handle without a comm is read in place, without the exchange.
 * comm == NULL: this process only.  comm != NULL: a collective call; every rank calls it with its own shards and every rank
 * gets the same outputs (each holds a replica of the coordinator's / learner's tallies; O(N) bytes cross ranks: 32 B per
 * Phase1b answer, 4 B per Phase2b answer).
 * RAPID_EINVAL, on every rank alike and before any answer moves, if: a shard is NULL or n_shards is outside [1, 64]; acceptor
 * ranges overlap; a shard has no answers of the wanted kind pending (last broadcast dropped for its configuration, or the
 * other phase); shards answered different broadcasts (rank, configuration or Phase2a value); a shard lives on a device other
 * than the px's.  A NULL px or a comm on another device than the px's is refused on that rank alone, without entering any
 * collective.  A refused call leaves the px unchanged. */
int32_t rapid_px_phase1b_from_acceptor_shards(rapid_px* px, const rapid_pxa* const* shards, int32_t n_shards, rapid_comm* comm,
                                              uint64_t perm_seed, int32_t* proposed, int64_t* trigger_index, uint64_t* cval_hash,
                                              uint64_t* cval_hash2, int32_t* cval_len, int64_t* n_messages);
int32_t rapid_px_phase2b_from_acceptor_shards(rapid_px* px, const rapid_pxa* const* shards, int32_t n_shards, rapid_comm* comm,
                                              uint64_t perm_seed, int32_t* decided, int64_t* decided_index, uint64_t* decided_hash,
                                              uint64_t* decided_hash2, int32_t* decided_len);
/* State of one acceptor: ranks[4] = rnd.round, rnd.node_index, vrnd.round, vrnd.node_index; its vval triple. */
int32_t rapid_pxa_read(const rapid_pxa* a, int64_t acceptor, int32_t* ranks, uint64_t* hash, uint64_t* hash2, int32_t* len);
/* Crashed processes never answer: acceptors with silent[r] != 0 (host array of n_acceptors bytes) change no state and send
 * nothing in rapid_pxa_phase1a / rapid_pxa_phase2a from now on.  silent == NULL clears the mask (every acceptor answers). */
int32_t rapid_pxa_set_silent(rapid_pxa* a, const uint8_t* silent);
/* *acceptor = the lowest local acceptor index whose vval is (hash, hash2, len), or -1 if none holds it.  A fast-round decision
 * is always some registered vote and a classic cval always some acceptor's vval, so called BEFORE rapid_pxa_phase2a overwrites
 * the vvals with the decided value this finds a proposer of it; with acceptors = detector receivers,
 * rapid_cd_get_proposal(that receiver) gives the value as ids. */
int32_t rapid_pxa_find_value(const rapid_pxa* a, uint64_t hash, uint64_t hash2, int32_t len, int64_t* acceptor);

/* ------------------------------------------------------------------------------------------------
 * Wire-format ingest  (rapid.proto; SURVEY.md §8 f3) — the step BEFORE the path: serialized protobuf bytes, as
 * they arrive at IMessagingServer / MembershipService.handleMessage(RapidRequest) (MembershipService.java:174),
 * straight into the cell SoA and the Endpoint -> id dictionary, on the device.
 * ---------------------------------------------------------------------------------------------- */
#define RAPID_WIRE_REQUEST 1u   /* the bytes are a RapidRequest (rapid.proto:21-35) whose content is the message */
/* A decoder owns the Endpoint{hostname, port} -> int32 id table of `v` (rebuilt when the view changes). */
int32_t rapid_wire_create(rapid_wire** out, rapid_view* v);
int32_t rapid_wire_destroy(rapid_wire* w);
/* The configuration the receiver is in: from now on only UP alerts carrying this configurationId register their edgeDst as a
 * joiner (a stale alert is dropped by filterAlertMessages, MembershipService.java:653, before it can introduce anything).
 * Without it every UP alert about an unknown endpoint registers one. */
int32_t rapid_wire_set_configuration(rapid_wire* w, int64_t cfg_id);
/* One serialized BatchedAlertMessage (rapid.proto:95-99): every AlertMessage (:101-110) becomes one cell per ring
 * number (MultiNodeCutDetector.java:79-80), in message order then ring order.  Endpoints map to ids; the edgeDst of
 * an UP alert that is not in the dictionary yet is REGISTERED as a joiner (rapid_view_register_joiners) in order of
 * first appearance; a DOWN alert about an unknown endpoint is dropped (MembershipService.java:660-664 would filter
 * it); an unknown edgeSrc becomes -1 (the detector never reads it).  Malformed bytes -> RAPID_EINVAL
 * (InvalidProtocolBufferException).  Unknown fields are skipped; packed and unpacked ringNumber are both accepted.
 * Outputs (each may be NULL): number of AlertMessages, cells produced, messages dropped, joiners registered, and
 * the id of BatchedAlertMessage.sender (-1 if unknown / absent). */
int32_t rapid_wire_decode_alerts(rapid_wire* w, const uint8_t* bytes, int64_t len, uint32_t flags, int64_t* n_messages,
                                 int64_t* n_cells, int64_t* n_dropped, int64_t* n_new_joiners, int32_t* sender_id);
/* The cells of the last decode, resident on the device (valid until the next decode on this handle): pass them to
 * rapid_cd_apply_batch_dev.  cfg carries each cell's AlertMessage.configurationId. */
int32_t rapid_wire_cells_dev(const rapid_wire* w, const int32_t** src, const int32_t** dst, const uint8_t** ring,
                             const uint8_t** status, const int64_t** cfg);
/* Host copies of the same (arrays of n_cells; each may be NULL). */
int32_t rapid_wire_read_cells(const rapid_wire* w, int32_t* src, int32_t* dst, uint8_t* ring, uint8_t* status, int64_t* cfg);
/* Per AlertMessage of the last decode (arrays of n_messages; each may be NULL): edgeDst id (-1 if dropped), edgeStatus,
 * number of ring numbers, NodeId (extractJoinerUuidAndMetadata, MembershipService.java:677-685; has_node_id = 0 if the
 * field is absent) and the byte range of the Metadata submessage inside the input buffer (len 0 if absent). */
int32_t rapid_wire_read_messages(const rapid_wire* w, int32_t* dst, uint8_t* status, int32_t* n_rings, int64_t* node_high,
                                 int64_t* node_low, uint8_t* has_node_id, int64_t* meta_off, int32_t* meta_len);
/* n serialized FastRoundPhase2bMessages (rapid.proto:105-110), message i = bytes[off[i] .. off[i+1]):
 * sender id (-1 if unknown), configurationId, and the proposal as rapid_proposal_fingerprint + size.  An endpoint that is
 * not in the dictionary (typical of a delayed vote of an earlier configuration, which FastPaxos.java:126-132 drops by its
 * configurationId) enters the fingerprint through its ring-0 key instead of an id: identical lists keep identical
 * fingerprints, nothing is refused, and rapid_fp_tally's configuration filter decides.  Proposal identity is
 * ORDER-INSENSITIVE (the Java compares List<Endpoint> in order; every proposer sorts by the ring-0 comparator first,
 * MembershipService.java:346-348, so well-formed votes never differ in order only). */
int32_t rapid_wire_decode_votes(rapid_wire* w, const uint8_t* bytes, const int64_t* off, int64_t n, uint32_t flags,
                                int32_t* sender, int64_t* vote_cfg, uint64_t* proposal_hash, uint64_t* proposal_hash2,
                                int32_t* proposal_len);
int32_t rapid_wire_last_device_ms(const rapid_wire* w, float* total_ms);

/* Consensus messages (rapid.proto:124-169).  A kind is the message's RapidRequest oneof case (rapid.proto:21-35). */
#define RAPID_WIRE_FAST_ROUND_PHASE2B 5   /* FastRoundPhase2bMessage {sender 1, configurationId 2, endpoints 3}          */
#define RAPID_WIRE_PHASE1A            6   /* Phase1aMessage {sender 1, configurationId 2, rank 3}                        */
#define RAPID_WIRE_PHASE1B            7   /* Phase1bMessage {sender 1, configurationId 2, rnd 3, vrnd 4, vval 5}         */
#define RAPID_WIRE_PHASE2A            8   /* Phase2aMessage {sender 1, configurationId 2, rnd 3, vval 5}                 */
#define RAPID_WIRE_PHASE2B            9   /* Phase2bMessage {sender 1, configurationId 2, rnd 3, endpoints 4}            */
/* n serialized messages of one kind, message i = bytes[off[i] .. off[i+1]) (off non-decreasing, within [0, 0x7ffffff0]).
 * With RAPID_WIRE_REQUEST each is a RapidRequest whose content must be the `kind` case: repeated occurrences of it merge,
 * another case occurring later replaces it, and a request whose content is not (or no longer) that case is malformed.
 * Per message, on the device: the sender id (-1 for an endpoint outside the dictionary, or an absent sender); the
 * configurationId; the rank — `rank` for Phase1a, `rnd` for Phase1b / 2a / 2b, (0, 0) for the fast round; `vrnd` for Phase1b,
 * else (0, 0); and the list as rapid_proposal_fingerprint of its ids plus its length.  Parsing follows the protobuf runtime:
 * proto3 defaults for absent fields (an absent Rank is (0, 0)), a repeated singular Rank or Endpoint is merged field by field,
 * an int32 is the low 32 bits of its varint, a field with an unexpected wire type and any unknown field is skipped (group
 * encodings, which rapid.proto never uses, are refused as malformed).  Malformed or truncated bytes give RAPID_EINVAL
 * ("malformed Phase1bMessage at index i", ...).
 * An endpoint outside the dictionary enters the fingerprint through its ring-0 key, exactly as in rapid_wire_decode_votes
 * (which is this decoder for kind 5): one list has one fingerprint whichever kind carries it, equal to the detector's
 * proposal fingerprint when every endpoint is known, so a value compares equal from fast-round vote to acceptor vval to
 * Phase1b, Phase2a and Phase2b.  Identity is ORDER-INSENSITIVE, as for votes: every well-formed value is a ring-0-sorted list
 * (MembershipService.java:346-348).  Outputs (may be NULL): messages whose sender is not in the dictionary, and list entries
 * that are not.  The decoded messages stay on the device for rapid_px_phase1b_wire / rapid_px_phase2b_wire /
 * rapid_fp_tally_wire.  Every decode on the handle (alerts included) replaces the last one; after a refused decode the
 * handle holds no consensus decode. */
int32_t rapid_wire_decode_consensus(rapid_wire* w, int32_t kind, const uint8_t* bytes, const int64_t* off, int64_t n,
                                    uint32_t flags, int64_t* n_unknown_senders, int64_t* n_unknown_endpoints);
/* Host copies of the per-message fields of the last consensus decode (arrays of n; each may be NULL). */
int32_t rapid_wire_read_consensus(const rapid_wire* w, int32_t* sender, int64_t* cfg, int32_t* rnd_round, int32_t* rnd_node,
                                  int32_t* vrnd_round, int32_t* vrnd_node, uint64_t* h1, uint64_t* h2, int32_t* len);
/* The list of message `index` of the last consensus decode as ids in wire order (-1 for an endpoint outside the dictionary):
 * writes min(cap, len) ids, *out_len = len.  Turns a trigger_index / decided_index back into a List<Endpoint>. */
int32_t rapid_wire_consensus_value(const rapid_wire* w, int64_t index, int32_t* out_ids, int32_t cap, int32_t* out_len);
/* The decoded messages of `w` handed to the tallies without leaving the device: rapid_px_phase1b / rapid_px_phase2b /
 * rapid_fp_tally over them in message order, same device code, same outputs; trigger / decided indexes are message indexes
 * of the decode.  RAPID_EINVAL, with the px / fp unchanged, if the last decode on w is not a successful decode of the
 * matching kind (Phase1b, Phase2b, FastRoundPhase2b), if w lives on another device, or (Phase2b and the fast round) if a
 * message OF THE CURRENT CONFIGURATION comes from an endpoint outside the dictionary.  Messages of another configuration are
 * dropped first, whatever their sender (Paxos.java:224, FastPaxos.java:126), so a delayed message from a node that has
 * since left is simply ignored.  The reference would count an unknown current-configuration sender as one more distinct
 * sender; members are the only senders in well-formed traffic, and collapsing unknown senders into one id would undercount
 * distinct senders, so the call is refused instead.  Phase1b never looks at its sender (handlePhase1bMessage appends). */
int32_t rapid_px_phase1b_wire(rapid_px* px, const rapid_wire* w, int32_t* proposed, int64_t* trigger_index, uint64_t* cval_hash,
                              uint64_t* cval_hash2, int32_t* cval_len, int64_t* n_messages);
int32_t rapid_px_phase2b_wire(rapid_px* px, const rapid_wire* w, int32_t* decided, int64_t* decided_index, uint64_t* decided_hash,
                              uint64_t* decided_hash2, int32_t* decided_len);
int32_t rapid_fp_tally_wire(rapid_fp* fp, const rapid_wire* w, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2,
                            int32_t* decided_len, int32_t* decided_count, int32_t* votes_received);

/* Wire-format egress: the messages the virtual nodes send, serialized on the device exactly as the protobuf runtime serializes
 * them (fields in field-number order, proto3 defaults omitted, a set submessage written even when empty, int32 / int64 values
 * sign-extended: a negative port, configurationId or NodeId half takes 10 bytes), each alone or (flags = RAPID_WIRE_REQUEST)
 * wrapped in a RapidRequest.  Message i = header i ++ body body_id[i] (no body when -1): the list-carrying kinds end with their
 * list, and every message that carries one list shares one copy of its bytes (the distinct (h1, h2, len) fingerprints).  The
 * encoder's outputs are the handle's own: a decode does not touch them nor an encode the last decode.  A refused encode
 * (RAPID_EINVAL, nothing written) leaves the previous encode's outputs as they were.
 *
 * One BatchedAlertMessage{sender, messages} per sender of the fdet's last interval (tick, then merge), senders in node order:
 * AlertMessage{edgeSrc = sender, edgeDst, edgeStatus, configurationId, ringNumber ascending and packed}, an UP (join) alert also
 * with nodeId = the joiner's NodeId (rapid_view_set_joiner_ids; zero halves if the view holds none) and an empty metadata, as
 * MembershipService.java:245-253 builds it; DOWN alerts as :486-492.  No bodies.  RAPID_EINVAL: fd created on another view or
 * device, or no interval since its reset (or the view changed since).  *n_bytes = all the bytes of the messages. */
int32_t rapid_wire_encode_alert_batches(rapid_wire* w, const rapid_fdet* fd, uint32_t flags, int64_t* n_messages, int64_t* n_bytes);
/* One FastRoundPhase2bMessage{sender, configurationId = cfg_id, endpoints} per receiver of cd that announced in its last call
 * (the receivers rapid_fp_tally_cd counts), in receiver order; receiver r's sender is the node at ring-0 position
 * receiver_begin + r, its endpoints its proposal in canonical ring-0 order (rapid_cd_get_proposal).  One body per distinct
 * proposal, numbered by its lowest receiver.  RAPID_EINVAL: cd created on another view or device, a RAW handle, or a handle that
 * has applied no batch yet or was created before the view's members last changed. */
int32_t rapid_wire_encode_votes(rapid_wire* w, const rapid_cd* cd, int64_t cfg_id, uint32_t flags, int64_t* n_messages, int64_t* n_bodies);
/* One Phase1bMessage{sender, configurationId, rnd, vrnd, vval} per answer of the acceptors' last rapid_pxa_phase1a / one
 * Phase2bMessage{sender, configurationId, rnd, endpoints} per answer of their last rapid_pxa_phase2a, as Paxos.java:136-142 /
 * :207-212 build them (rnd and vrnd always set), in acceptor order; silent acceptors and those that did not answer send nothing.
 * Acceptor g (acceptor_begin + local index) is the node at ring-0 position g of w's view, as a detector receiver is.  An empty
 * vval has no body.  Each distinct list is taken from the lists this handle fetched before in the same membership (the votes it
 * encoded: every registered vote and every Phase2a value is some announced proposal), else from the announced proposal of
 * receiver g - receiver_begin of cd (may be NULL), which must match the list's fingerprint.  RAPID_EINVAL, nothing written: no
 * answers of that kind pending, acceptors on another device or beyond the view, cd on another view / device / membership, or a
 * list found in neither place. */
int32_t rapid_wire_encode_phase1b(rapid_wire* w, const rapid_pxa* pxa, const rapid_cd* cd, uint32_t flags, int64_t* n_messages,
                                  int64_t* n_bodies);
int32_t rapid_wire_encode_phase2b(rapid_wire* w, const rapid_pxa* pxa, const rapid_cd* cd, uint32_t flags, int64_t* n_messages,
                                  int64_t* n_bodies);
/* The last encode: messages, header bytes, bodies, body bytes (all 0 before the first encode). */
int32_t rapid_wire_encoded_counts(const rapid_wire* w, int64_t* n_messages, int64_t* header_bytes, int64_t* n_bodies, int64_t* body_bytes);
/* Its outputs on the device (valid until the next encode on the handle) / host copies: headers[header_bytes],
 * header_off[n_messages + 1], body_id[n_messages], bodies[body_bytes], body_off[n_bodies + 1].  Each may be NULL. */
int32_t rapid_wire_encoded_dev(const rapid_wire* w, const uint8_t** headers, const int64_t** header_off, const int32_t** body_id,
                               const uint8_t** bodies, const int64_t** body_off);
int32_t rapid_wire_read_encoded(const rapid_wire* w, uint8_t* headers, int64_t* header_off, int32_t* body_id, uint8_t* bodies,
                                int64_t* body_off);
/* sizes[n_messages]: the whole size of every message, header + body, computed on the device. */
int32_t rapid_wire_read_encoded_sizes(const rapid_wire* w, int64_t* sizes);
/* sender[n_messages]: the view id of every message's sender. */
int32_t rapid_wire_read_encoded_senders(const rapid_wire* w, int32_t* sender);

/* ------------------------------------------------------------------------------------------------
 * Alert generation  (SURVEY.md §8 f4): PingPongFailureDetector.java:38-121 — one detector per entry of
 * getSubjectsOf(node), i.e. K per member (MembershipService.java:697-707) — and the AlertMessage a notifier
 * raises (edgeFailureNotification, MembershipService.java:472-495: DOWN, every ring number of the edge).
 * The network is a scenario: per-node flags and optional per-detector probe failures.
 * ---------------------------------------------------------------------------------------------- */
#define RAPID_FD_CRASHED         1u   /* answers no probe and runs no detector                               */
#define RAPID_FD_INGRESS_BLOCKED 2u   /* probes TO the node fail                                             */
#define RAPID_FD_EGRESS_BLOCKED  4u   /* probes FROM the node fail                                           */
#define RAPID_FD_BOOTSTRAPPING   8u   /* answers NodeStatus.BOOTSTRAPPING (tolerated bootstrap_threshold times, :45, :97-104) */
/* failure_threshold = FAILURE_THRESHOLD (10, :41), bootstrap_threshold = BOOTSTRAP_COUNT_THRESHOLD (30, :45). */
int32_t rapid_fdet_create(rapid_fdet** out, const rapid_view* v, int32_t failure_threshold, int32_t bootstrap_threshold);
int32_t rapid_fdet_destroy(rapid_fdet* fd);
/* New configuration: cancelFailureDetectorJobs + createFailureDetectorsForCurrentConfiguration (MembershipService.java:433-434). */
int32_t rapid_fdet_reset(rapid_fdet* fd);
/* One failure-detector interval of every live node: run() (:75-85) of its K detectors in ring order — notify if
 * failureCount >= threshold and not yet notified, else probe and count a failure (:120-123).  node_flags[n]: RAPID_FD_* of
 * every member; edge_fail[n * K] (may be NULL): non-zero = the probe of that node's k-th detector fails regardless.
 * The notifications of this interval become AlertMessages{edgeSrc = node, edgeDst = subject, DOWN, cfg_id, all ring numbers
 * of the edge} and their cells, ordered by node id, then detector, then ring number; they stay on the device. */
int32_t rapid_fdet_tick(rapid_fdet* fd, const uint8_t* node_flags, const uint8_t* edge_fail, int64_t cfg_id, int64_t* n_alerts,
                        int64_t* n_cells);
int32_t rapid_fdet_tick_dev(rapid_fdet* fd, const uint8_t* node_flags_dev, const uint8_t* edge_fail_dev, int64_t cfg_id,
                            int64_t* n_alerts, int64_t* n_cells);
/* Cells of the last tick on the device (for rapid_cd_apply_batch_dev) / on the host; alerts as (observer, subject, ring bitmask). */
int32_t rapid_fdet_cells_dev(const rapid_fdet* fd, const int32_t** src, const int32_t** dst, const uint8_t** ring,
                             const uint8_t** status, const int64_t** cfg);
/* The last interval's cells grouped as the reference ships them — AlertBatcher sends ONE BatchedAlertMessage per sender and
 * window (MembershipService.java:613-637): batch b = the cells raised by one observer.  batch_off[0 .. *n_batches] feeds
 * rapid_cd_apply_batches_dev together with rapid_fdet_cells_dev; RAPID_ENOMEM (with *n_batches set) if cap is too small. */
int32_t rapid_fdet_sender_batches(const rapid_fdet* fd, int64_t* batch_off, int64_t cap, int64_t* n_batches);
/* Join phase 2 (MembershipService.java:232-281) in the interval of the last tick: for every listed registered joiner j (host
 * array of view ids), each of its K expected observers o (predecessors of j on the rings) that is not RAPID_FD_CRASHED in that
 * tick's node flags raises ONE AlertMessage{edgeSrc = o, edgeDst = j, UP, cfg_id, ring numbers = {k : observer k of j is o}}.
 * They join the interval's alerts and cells, re-ordered so that every sender's alerts stay contiguous: by sender, the
 * detectors' alerts first (tick order), then the join alerts in the order the joiners are listed.  rapid_fdet_sender_batches,
 * rapid_fdet_cells_dev and rapid_fdet_read_* then describe the merged interval.  An id that is not a registered joiner gives
 * RAPID_EINVAL and leaves the interval as the tick made it.  One call per tick: a second call before the next tick gives
 * RAPID_EINVAL and changes nothing (list every joiner of the interval in one call).  *n_alerts / *n_cells: totals of the
 * merged interval.  After rapid_fdet_tick_dev the caller's node_flags_dev must still hold that tick's flags.
 * Same as rapid_fdet_merge_alerts(fd, joiner_ids, n, NULL, 0, cfg_id, n_alerts, n_cells). */
int32_t rapid_fdet_join_alerts(rapid_fdet* fd, const int32_t* joiner_ids, int64_t n, int64_t cfg_id, int64_t* n_alerts,
                               int64_t* n_cells);
/* Join and leave alerts merged into the interval of the last tick, in one call.
 * Join candidates: as rapid_fdet_join_alerts (UP, one alert per distinct live expected observer).
 * Leave candidates (MembershipService.leave :545-565 -> handleLeaveMessage :372-376 -> edgeFailureNotification :472-495): for
 * every listed member l (host array of view ids) and every k in 0..K-1, o = observer k of l (getObserversOf, the obs row of l)
 * raises one AlertMessage{edgeSrc = o, edgeDst = l, DOWN, cfg_id, ring numbers = {r : observer r of l is o}} unless o is
 * RAPID_FD_CRASHED in the tick's node flags.  Repeats are kept, as the reference sends one LeaveMessage per entry of
 * getObserversOf: an observer on m rings of l raises m identical alerts, so a leaver whose observers all live raises K alerts
 * and sum_o m_o^2 cells.  The leaver's own flags are not read (it has shut down; callers mark it crashed in the same tick).
 * Only RAPID_FD_CRASHED silences an observer.  In a view of fewer than 2 members a leave raises nothing (:240-242).
 * Order per sender: the tick's alerts (tick order), then the join alerts (list order), then the leave alerts (list order, then
 * k).  RAPID_EINVAL, with the interval exactly as the tick made it: an id that is not a registered joiner (joiner_ids) or not a
 * member (leaver_ids), 2^30 or more candidates (tick alerts + K per listed id), a view changed since the tick, no tick yet, or
 * a second merge into the same interval ("already added", whichever kinds the first call carried).  An accepted merge sets
 * rapid_fdet_last_device_ms to its own device time (0 if it launched nothing). */
int32_t rapid_fdet_merge_alerts(rapid_fdet* fd, const int32_t* joiner_ids, int64_t n_joiners, const int32_t* leaver_ids,
                                int64_t n_leavers, int64_t cfg_id, int64_t* n_alerts, int64_t* n_cells);
int32_t rapid_fdet_read_cells(const rapid_fdet* fd, int32_t* src, int32_t* dst, uint8_t* ring, uint8_t* status, int64_t* cfg);
int32_t rapid_fdet_read_alerts(const rapid_fdet* fd, int32_t* observer, int32_t* subject, uint16_t* ring_mask);
/* failureCount / notified of node's k-th detector */
int32_t rapid_fdet_state(const rapid_fdet* fd, int64_t node, int32_t k, int32_t* failure_count, int32_t* notified);
int32_t rapid_fdet_last_device_ms(const rapid_fdet* fd, float* total_ms);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU; receivers sharded by ring-0 range; one all-reduce on the histogram)
 * ---------------------------------------------------------------------------------------------- */
#define RAPID_NCCL_UNIQUE_ID_BYTES 128
int32_t rapid_comm_unique_id(void* out_id /*128 bytes*/);
int32_t rapid_comm_init(rapid_comm** out, int32_t rank, int32_t world, const void* nccl_unique_id, int32_t device);
int32_t rapid_comm_destroy(rapid_comm* c);

/* Timing aid for bench.py: device time (ms) of the last rapid_cd_apply_batch[_dev] / rapid_fp_tally[_cd] call,
 * measured with CUDA events on the handle's stream; and per-kernel breakdown of the last apply. */
int32_t rapid_cd_last_device_ms(const rapid_cd* cd, float* total_ms, float* main_kernel_ms);
int32_t rapid_fp_last_device_ms(const rapid_fp* fp, float* total_ms);
int32_t rapid_fp_last_launches(const rapid_fp* fp, int32_t* n_kernel_launches);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* RAPID_B200_H */
