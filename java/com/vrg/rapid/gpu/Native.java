/*
 * JNI veneer over librapid_b200.so (include/rapid_b200.h).  UNCOMPILED in this repository's build image (no JDK);
 * it is the binding a Rapid maintainer adds: one static native per C entry point, handles as long, arrays as direct
 * ByteBuffers / primitive arrays.  Every method returns the C status code (0 ok, <0 error); lastError() is the message.
 */
package com.vrg.rapid.gpu;

import java.nio.ByteBuffer;

public final class Native {
    static {
        System.loadLibrary("rapid_jni");     // java/jni/rapid_jni.c, linked against librapid_b200.so
    }

    private Native() {
    }

    public static native String lastError();

    // ---- MembershipView (com.vrg.rapid.MembershipView) ----
    /** rapid_view_create: hostBytes = hostnames concatenated, hostOff[n+1]; returns handle or 0 (see lastError). */
    public static native long viewCreate(int k, long n, byte[] hostBytes, int[] hostOff, int[] port, int device);
    public static native int viewDestroy(long view);
    public static native int viewRing(long view, int ring, int[] outIds);
    public static native int viewObservers(long view, int node, int[] outK);          // returns count or <0
    public static native int viewSubjects(long view, int node, int[] outK);
    public static native int viewExpectedObservers(long view, byte[] host, int port, int[] outK);
    public static native int viewRingNumbers(long view, int observer, int subject);   // bitmask or <0
    public static native int viewConfigId(long view, long[] idHigh, long[] idLow, long[] out1);
    public static native int viewRegisterJoiners(long view, byte[] hostBytes, int[] hostOff, int[] port);  // first id
    /** decideViewChange on the device (rapid_view_apply_cut): members in the cut leave, registered joiners in it are added;
     *  outOldToNew may be null.  RAPID_EUUID_SEEN (-4) = UUIDAlreadySeenException, nothing changed. */
    public static native int viewApplyCut(long view, int[] cutIds, int[] outOldToNew);
    /** identifiersSeen on the device: NodeIds of the members (index = node id) / of registered joiners */
    public static native int viewSetNodeIds(long view, long[] idHigh, long[] idLow);
    public static native int viewSetJoinerIds(long view, int firstJoinerId, long[] idHigh, long[] idLow);
    /** getCurrentConfigurationId from the device-resident identifiersSeen + ring 0 */
    public static native int viewCurrentConfigId(long view, long[] out1);
    /** rapid_view_overlay_spectrum: tolBits = Double.doubleToRawLongBits(tol); out5 = raw bits of lambda2, lambda_min and residual
     *  (Double.longBitsToDouble), the steps spent, raw bits of the device milliseconds (as a double). */
    public static native int viewOverlaySpectrum(long view, long seed, long tolBits, int maxSteps, long[] out5);

    // ---- MultiNodeCutDetector / alert-batch handler ----
    public static native long cdCreate(long view, int h, int l, long receivers, long receiverBegin, int modeFlags,
                                       long maxSubjects);
    public static native int cdDestroy(long cd);
    /** rapid_cd_apply_batch with direct buffers: dst int32[n], ring uint8[n], status uint8[n]; outputs may be null. */
    public static native int cdApplyBatch(long cd, long cfgId, long nCells, ByteBuffer dst, ByteBuffer ring,
                                          ByteBuffer status, ByteBuffer cellCfg, int deliveryFlags, ByteBuffer blocked,
                                          ByteBuffer bitmap, long permSeed, ByteBuffer outHash, ByteBuffer outHash2,
                                          ByteBuffer outLen, ByteBuffer outAnnounced);
    public static native int cdGetProposal(long cd, long receiver, int[] outIds);      // returns length or <0
    /** rapid_cd_proposal_census: the distinct proposals announced in the detector's last call (VIEW_CHANGE_PROPOSAL's payload,
     *  one NodeStatusChange list per class).  cutIds may be null; out2 = {classes, entries}. */
    public static native int cdProposalCensus(long cd, int[] cutIds, long[] out2);
    /** rapid_cd_read_census into direct buffers (any may be null): hash, hash2 uint64[classes], len, voters, representative,
     *  inCut int32[classes], listOff int64[classes + 1], ids int32[entries], status uint8[entries] (0 = UP, 1 = DOWN) */
    public static native int cdReadCensus(long cd, ByteBuffer hash, ByteBuffer hash2, ByteBuffer len, ByteBuffer voters,
                                          ByteBuffer representative, ByteBuffer inCut, ByteBuffer listOff, ByteBuffer ids,
                                          ByteBuffer status);
    /** class of every receiver of the last census, -1 = did not announce */
    public static native int cdReadCensusClasses(long cd, int[] cls);
    public static native int cdAggregate(long cd, int[] dst, byte[] ring, byte[] status, long receiver, int[] outIds);
    public static native int cdInvalidate(long cd, long receiver, int[] outIds);
    public static native int cdNumProposals(long cd, long receiver);
    public static native int cdClear(long cd);
    /** out4 = {sequences served in one pass, replayed batch by batch, receivers failing premise A1 / A2 in the last refusal} */
    public static native int cdSequenceStats(long cd, int[] out4);
    /** wait for asynchronous batches (wireApplyToDetector / fdetApplyToDetector with async = true); returns their latched status */
    public static native int cdSync(long cd);
    /** several BatchedAlertMessages in one call: batch b = cells [batchOff[b], batchOff[b+1]); announcedIn[r] = batch index or -1 */
    public static native int cdApplyBatches(long cd, long cfgId, int[] dst, byte[] ring, byte[] status, long[] cellCfg, long[] batchOff,
                                            ByteBuffer outHash, ByteBuffer outHash2, ByteBuffer outLen, ByteBuffer outAnnounced,
                                            ByteBuffer outAnnouncedIn);

    // ---- FastPaxos fast round ----
    public static native long fpCreate(long cfgId, long membershipSize, long senderCapacity, int device);
    public static native int fpDestroy(long fp);
    public static native int fpReset(long fp, long cfgId, long membershipSize);
    /** out6 = {decided, hashLo.. } see rapid_fp_tally; returns status */
    public static native int fpTally(long fp, int[] sender, long[] voteCfg, long[] hash, long[] hash2, int[] len,
                                     long[] out6);
    public static native int fpTallyCd(long fp, long cd, long comm, long[] out6);
    /** enqueue only (rapid_fp_tally_cd_async) / collect the last enqueued tally: out7 = out6 + {decidedInCall} */
    public static native int fpTallyCdAsync(long fp, long cd, long comm);
    public static native int fpResult(long fp, long[] out7);

    public static native long[] proposalFingerprint(int[] ids);

    // ---- classic Paxos fallback (Paxos.java) ----
    public static native long pxCreate(long cfgId, long membershipSize, long messageCapacity, int device);
    public static native int pxDestroy(long px);
    /** startPhase1a: returns 1 if crnd moved to (round, nodeIndex), 0 if ignored, <0 status */
    public static native int pxStartPhase1a(long px, int round, int nodeIndex);
    /** selectProposalUsingCoordinatorRule: index of the message whose vval is chosen, -1 = empty list, <-1 status-2 */
    public static native long pxCoordinatorRule(long px, int[] vrndRound, int[] vrndNode, long[] hash, long[] hash2, int[] len);
    /** handlePhase1bMessage over a batch; out6 = {proposed, triggerIndex, cvalHash, cvalHash2, cvalLen, nMessages} */
    public static native int pxPhase1b(long px, long[] msgCfg, int[] rndRound, int[] rndNode, int[] vrndRound, int[] vrndNode,
                                       long[] hash, long[] hash2, int[] len, long[] out6);
    /** handlePhase2bMessage over a batch; out5 = {decided, decidedIndex, hash, hash2, len} */
    public static native int pxPhase2b(long px, long[] msgCfg, int[] rndRound, int[] rndNode, int[] sender, long[] hash,
                                       long[] hash2, int[] len, long[] out5);
    public static native long pxaCreate(long cfgId, long nAcceptors, long acceptorBegin, int device);
    public static native int pxaDestroy(long pxa);
    public static native int pxaRegisterFastRoundVotesCd(long pxa, long cd);
    public static native long pxaPhase1a(long pxa, long msgCfg, int round, int nodeIndex);            // replies or <0
    public static native long pxaPhase2a(long pxa, long msgCfg, int round, int nodeIndex, long hash, long hash2, int len);
    /** the answers of the last pxaPhase1a / pxaPhase2a of this rank's acceptor shards (and, comm != 0, every rank's: a
     *  collective call), delivered to the tallies; one shard, comm == 0: a single handle; out6 / out5 as pxPhase1b / pxPhase2b */
    public static native int pxPhase1bFromAcceptorShards(long px, long[] pxaShards, long comm, long permSeed, long[] out6);
    public static native int pxPhase2bFromAcceptorShards(long px, long[] pxaShards, long comm, long permSeed, long[] out5);

    // ---- wire-format ingest (rapid.proto bytes -> cells on the device) ----
    public static native long wireCreate(long view);
    /** only UP alerts of this configuration register joiners from now on */
    public static native int wireSetConfiguration(long wire, long cfgId);
    public static native int wireDestroy(long wire);
    /** bytes = BatchedAlertMessage.toByteArray() (or the RapidRequest, asRequest); out5 = {nMessages, nCells, nDropped, nNewJoiners, senderId} */
    public static native int wireDecodeAlerts(long wire, ByteBuffer bytes, int len, boolean asRequest, long[] out5);
    /** apply the cells of the last decode to a detector without leaving the device (rapid_wire_cells_dev + rapid_cd_apply_batch_dev) */
    public static native int wireApplyToDetector(long wire, long cd, long cfgId, long nCells);
    /** same, enqueue only (rapid_cd_apply_batch_dev_async): the status comes back from cdSync / fpTallyCd */
    public static native int wireApplyToDetectorAsync(long wire, long cd, long cfgId, long nCells);
    /** consensus messages of one kind (5 FastRoundPhase2b, 6 Phase1a, 7 Phase1b, 8 Phase2a, 9 Phase2b; each message's bytes
     *  are bytes[off[i] .. off[i+1]), the RapidRequest when asRequest) decoded on the device; out2 = {unknown senders,
     *  unknown list entries} */
    public static native int wireDecodeConsensus(long wire, int kind, ByteBuffer bytes, long[] off, boolean asRequest, long[] out2);
    /** per message of the last consensus decode (arrays of n, each may be null) */
    public static native int wireReadConsensus(long wire, int[] sender, long[] cfg, int[] rndRound, int[] rndNode, int[] vrndRound,
                                               int[] vrndNode, long[] hash, long[] hash2, int[] len);
    /** the list of message `index` as ids in wire order (-1 = not in the view); returns its length or <0; fills min(len, outIds.length) */
    public static native int wireConsensusValue(long wire, long index, int[] outIds);
    /** handlePhase1bMessage / handlePhase2bMessage / handleFastRoundProposal over the last decode, without leaving the device;
     *  outputs as pxPhase1b (out6), pxPhase2b (out5), fpTally (out6) */
    public static native int pxPhase1bWire(long px, long wire, long[] out6);
    public static native int pxPhase2bWire(long px, long wire, long[] out5);
    public static native int fpTallyWire(long fp, long wire, long[] out6);

    // ---- wire-format egress (the virtual nodes' messages -> rapid.proto bytes, encoded on the device) ----
    /** one BatchedAlertMessage per sender of the fdet's last interval; out2 = {nMessages, nBytes} */
    public static native int wireEncodeAlertBatches(long wire, long fdet, boolean asRequest, long[] out2);
    /** one FastRoundPhase2bMessage per receiver of cd that announced in its last call; out2 = {nMessages, nBodies} */
    public static native int wireEncodeVotes(long wire, long cd, long cfgId, boolean asRequest, long[] out2);
    /** one Phase1bMessage / Phase2bMessage per answer of the pxa's last Phase1a / Phase2a; lists from the votes encoded before, else
     *  from cd's receivers (cd may be 0); out2 = {nMessages, nBodies} */
    public static native int wireEncodePhase1b(long wire, long pxa, long cd, boolean asRequest, long[] out2);
    public static native int wireEncodePhase2b(long wire, long pxa, long cd, boolean asRequest, long[] out2);
    /** the view id of every message's sender */
    public static native int wireReadEncodedSenders(long wire, int[] sender);
    /** the last encode: out4 = {nMessages, headerBytes, nBodies, bodyBytes} */
    public static native int wireEncodedCounts(long wire, long[] out4);
    /** its device pointers: out5 = {headers, headerOff, bodyId, bodies, bodyOff} */
    public static native int wireEncodedDev(long wire, long[] out5);
    /** host copies (each may be null): message i = headers[headerOff[i] .. headerOff[i+1]) ++ body bodyId[i] (none if -1) */
    public static native int wireReadEncoded(long wire, byte[] headers, long[] headerOff, int[] bodyId, byte[] bodies, long[] bodyOff);
    /** bytes of every message of the last encode, header + body */
    public static native int wireReadEncodedSizes(long wire, long[] sizes);

    // ---- alert generation: the K PingPongFailureDetectors of every virtual node ----
    public static native long fdetCreate(long view, int failureThreshold, int bootstrapThreshold);
    public static native int fdetDestroy(long fdet);
    public static native int fdetReset(long fdet);
    /** one failure-detector interval; out2 = {nAlerts, nCells}; the cells stay on the device */
    public static native int fdetTick(long fdet, byte[] nodeFlags, byte[] edgeFail, long cfgId, long[] out2);
    public static native int fdetApplyToDetector(long fdet, long cd, long cfgId, long nCells);
}
