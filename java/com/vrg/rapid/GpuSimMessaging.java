/*
 * Seam 2 of INTEGRATION.md: a virtual cluster behind Rapid's messaging SPI.  UNCOMPILED here (no JDK).
 *
 * implements IMessagingClient (messaging/IMessagingClient.java:25-49) and IMessagingServer (:24-41): instead of a socket,
 * sendMessageBestEffort(remote, BATCHEDALERTMESSAGE) applies the batch to the HBM-resident detectors of every virtual
 * node (UnicastToAllBroadcaster.java:46-52 sends the same request to all members: the first unicast of a broadcast
 * triggers the device call, the rest are no-ops), and FASTROUNDPHASE2BMESSAGE votes are tallied on the device.  One mutex
 * serialises callers (protocol thread / "msbg" batcher thread, MembershipService.java:630).
 *
 * Return path: what the virtual nodes send back is encoded on the device (rapid_wire_encode_*) and handed to the real node's
 * MembershipService as RapidRequests: the votes of the virtual nodes that announced after each batch, the Phase1b / Phase2b
 * answers of the virtual acceptors to the real node's Phase1a / Phase2a, and (deliverVirtualAlerts) the alert batches of a
 * device failure-detector interval.  Every broadcast reaches every member, the real node included.
 */
package com.vrg.rapid;

import com.google.common.util.concurrent.Futures;
import com.google.common.util.concurrent.ListenableFuture;
import com.vrg.rapid.gpu.Native;
import com.vrg.rapid.messaging.IMessagingClient;
import com.vrg.rapid.messaging.IMessagingServer;
import com.vrg.rapid.pb.AlertMessage;
import com.vrg.rapid.pb.BatchedAlertMessage;
import com.google.protobuf.ByteString;
import com.google.protobuf.InvalidProtocolBufferException;
import com.vrg.rapid.pb.Endpoint;
import com.vrg.rapid.pb.Phase1aMessage;
import com.vrg.rapid.pb.Phase2aMessage;
import com.vrg.rapid.pb.RapidRequest;
import com.vrg.rapid.pb.RapidResponse;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;

final class GpuSimMessaging implements IMessagingClient, IMessagingServer {
    private final Object lock = new Object();
    private final GpuMembershipView view;
    private final long cd;
    private final long fp;
    private final long pxa;
    private final long wire;
    private final long configurationId;
    private BatchedAlertMessage lastApplied;      // identity of the broadcast already applied
    private Phase1aMessage lastPhase1a;
    private Phase2aMessage lastPhase2a;
    private MembershipService service;            // the real node, which receives the virtual nodes' messages

    GpuSimMessaging(final GpuMembershipView view, final long configurationId, final int H, final int L,
                    final int members) {
        this.view = view;
        this.configurationId = configurationId;
        this.cd = Native.cdCreate(view.handle(), H, L, members, 0, 0 /* SERVICE, bucketed */, 0);
        this.fp = Native.fpCreate(configurationId, members, members, 0);
        this.pxa = Native.pxaCreate(configurationId, members, 0, 0);   // acceptor r = receiver r = ring-0 position r
        this.wire = Native.wireCreate(view.handle());
    }

    @Override
    public ListenableFuture<RapidResponse> sendMessageBestEffort(final Endpoint remote, final RapidRequest msg) {
        synchronized (lock) {
            switch (msg.getContentCase()) {
                case BATCHEDALERTMESSAGE:
                    if (msg.getBatchedAlertMessage() != lastApplied) {   // one device call per broadcast
                        lastApplied = msg.getBatchedAlertMessage();
                        applyBatch(lastApplied);
                        final long[] out = new long[6];
                        Native.fpTallyCd(fp, cd, 0, out);                // every virtual node that announced votes
                        Native.pxaRegisterFastRoundVotesCd(pxa, cd);
                        final long[] out2 = new long[2];
                        if (Native.wireEncodeVotes(wire, cd, configurationId, true, out2) == 0) {
                            deliver();                                   // ... and the real node receives their votes
                        }
                    }
                    break;
                case PHASE1AMESSAGE:
                    if (msg.getPhase1aMessage() != lastPhase1a) {
                        lastPhase1a = msg.getPhase1aMessage();
                        Native.pxaPhase1a(pxa, lastPhase1a.getConfigurationId(), lastPhase1a.getRank().getRound(),
                                          lastPhase1a.getRank().getNodeIndex());
                        final long[] out2 = new long[2];
                        if (Native.wireEncodePhase1b(wire, pxa, cd, true, out2) == 0) {
                            deliver();
                        }
                    }
                    break;
                case PHASE2AMESSAGE:
                    if (msg.getPhase2aMessage() != lastPhase2a) {
                        lastPhase2a = msg.getPhase2aMessage();
                        final int[] ids = new int[lastPhase2a.getVvalCount()];
                        for (int i = 0; i < ids.length; i++) {
                            ids[i] = view.idOf(lastPhase2a.getVval(i), false);
                        }
                        final long[] h = Native.proposalFingerprint(ids);
                        Native.pxaPhase2a(pxa, lastPhase2a.getConfigurationId(), lastPhase2a.getRnd().getRound(),
                                          lastPhase2a.getRnd().getNodeIndex(), h[0], h[1], ids.length);
                        final long[] out2 = new long[2];
                        if (Native.wireEncodePhase2b(wire, pxa, cd, true, out2) == 0) {
                            deliver();
                        }
                    }
                    break;
                default:
                    break;                                               // probes, joins: not simulated on the device
            }
        }
        return Futures.immediateFuture(RapidResponse.getDefaultInstance());
    }

    /** the alert batches of the last interval of a device failure detector (rapid_fdet) created on the same view */
    void deliverVirtualAlerts(final long fdet) {
        synchronized (lock) {
            final long[] out2 = new long[2];
            if (Native.wireEncodeAlertBatches(wire, fdet, true, out2) == 0) {
                deliver();
            }
        }
    }

    // The last encode as RapidRequests to the real node: header i ++ body bodyId[i]; ByteString.concat shares a body's bytes
    // between the messages that carry it instead of copying them per message.
    private void deliver() {
        if (service == null) {
            return;
        }
        final long[] counts = new long[4];
        Native.wireEncodedCounts(wire, counts);
        final int n = (int) counts[0];
        final byte[] headers = new byte[(int) counts[1]];
        final long[] headerOff = new long[n + 1];
        final int[] bodyId = new int[n];
        final byte[] bodies = new byte[(int) counts[3]];
        final long[] bodyOff = new long[(int) counts[2] + 1];
        if (Native.wireReadEncoded(wire, headers, headerOff, bodyId, bodies, bodyOff) != 0) {
            return;
        }
        final ByteString[] body = new ByteString[(int) counts[2]];
        for (int b = 0; b < body.length; b++) {
            body[b] = ByteString.copyFrom(bodies, (int) bodyOff[b], (int) (bodyOff[b + 1] - bodyOff[b]));
        }
        for (int i = 0; i < n; i++) {
            ByteString m = ByteString.copyFrom(headers, (int) headerOff[i], (int) (headerOff[i + 1] - headerOff[i]));
            if (bodyId[i] >= 0) {
                m = m.concat(body[bodyId[i]]);
            }
            try {
                service.handleMessage(RapidRequest.parseFrom(m));
            } catch (final InvalidProtocolBufferException e) {
                throw new IllegalStateException("the device encoded a malformed RapidRequest", e);
            }
        }
    }

    private void applyBatch(final BatchedAlertMessage batch) {
        int cells = 0;
        for (final AlertMessage m : batch.getMessagesList()) {
            cells += m.getRingNumberCount();
        }
        final ByteBuffer dst = ByteBuffer.allocateDirect(4 * cells).order(ByteOrder.nativeOrder());
        final ByteBuffer ring = ByteBuffer.allocateDirect(cells);
        final ByteBuffer status = ByteBuffer.allocateDirect(cells);
        final ByteBuffer cfg = ByteBuffer.allocateDirect(8 * cells).order(ByteOrder.nativeOrder());
        for (final AlertMessage m : batch.getMessagesList()) {
            final int id = view.idOf(m.getEdgeDst(), true);
            for (int i = 0; i < m.getRingNumberCount(); i++) {       // one cell per ring number (MultiNodeCutDetector.java:79-80)
                dst.putInt(id);
                ring.put((byte) m.getRingNumber(i));
                status.put((byte) m.getEdgeStatusValue());
                cfg.putLong(m.getConfigurationId());
            }
        }
        Native.cdApplyBatch(cd, configurationId, cells, dst, ring, status, cfg, 0, null, null, 0L, null, null, null, null);
    }

    @Override
    public ListenableFuture<RapidResponse> sendMessage(final Endpoint remote, final RapidRequest msg) {
        return sendMessageBestEffort(remote, msg);
    }

    @Override
    public void start() {
    }

    @Override
    public void shutdown() {
        Native.wireDestroy(wire);
        Native.pxaDestroy(pxa);
        Native.cdDestroy(cd);
        Native.fpDestroy(fp);
    }

    @Override
    public void setMembershipService(final MembershipService service) {
        synchronized (lock) {
            this.service = service;
        }
    }
}
