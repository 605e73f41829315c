/*
 * Read side of com.vrg.rapid.MembershipView served from the device-resident K-ring view.  UNCOMPILED here (no JDK).
 * Built once per configuration from the full endpoint list (ring mutations stay in the Java view, which the service
 * keeps for the join protocol); ids: members 0..n-1 in list order, joiners registered afterwards.
 */
package com.vrg.rapid;

import com.vrg.rapid.gpu.Native;
import com.vrg.rapid.pb.Endpoint;

import java.io.ByteArrayOutputStream;
import java.util.ArrayList;
import java.util.HashMap;
import java.util.List;
import java.util.Map;

final class GpuMembershipView {
    private final int K;
    private final long handle;
    private final List<Endpoint> byId = new ArrayList<>();
    private final Map<Endpoint, Integer> ids = new HashMap<>();
    private int members;

    GpuMembershipView(final int K, final List<Endpoint> endpoints, final int device) {
        this.K = K;
        final ByteArrayOutputStream bytes = new ByteArrayOutputStream();
        final int[] off = new int[endpoints.size() + 1];
        final int[] port = new int[endpoints.size()];
        int i = 0;
        for (final Endpoint e : endpoints) {
            final byte[] h = e.getHostname().toByteArray();
            bytes.write(h, 0, h.length);
            off[i + 1] = off[i] + h.length;
            port[i] = e.getPort();
            ids.put(e, i);
            byId.add(e);
            i++;
        }
        this.members = endpoints.size();
        this.handle = Native.viewCreate(K, members, bytes.toByteArray(), off, port, device);
        if (handle == 0) {
            throw new IllegalStateException(Native.lastError());
        }
    }

    long handle() {
        return handle;
    }

    boolean isHostPresent(final Endpoint e) {                 // MembershipView.java:330-337
        final Integer id = ids.get(e);
        return id != null && id < members;
    }

    int idOf(final Endpoint e, final boolean registerAsJoiner) {
        Integer id = ids.get(e);
        if (id == null) {
            if (!registerAsJoiner) {
                throw new MembershipView.NodeNotInRingException(e);
            }
            final byte[] h = e.getHostname().toByteArray();
            id = Native.viewRegisterJoiners(handle, h, new int[]{0, h.length}, new int[]{e.getPort()});
            ids.put(e, id);
            byId.add(e);
        }
        return id;
    }

    Endpoint endpointOf(final int id) {
        return byId.get(id);
    }


    /**
     * decideViewChange (MembershipService.java:385-444) on the device: the members named by the decision leave (ringDelete
     * :167-201), the joiners named by it — registered when their UP alerts arrived — are added (ringAdd :123-160).  The K rings
     * are updated in HBM (compaction + sorted merge); only the cut's ids go down and the id mapping comes back.
     */
    void applyViewChange(final List<Endpoint> decidedCut) {
        final int[] cut = new int[decidedCut.size()];
        for (int i = 0; i < cut.length; i++) {
            cut[i] = idOf(decidedCut.get(i), false);
        }
        final int[] oldToNew = new int[byId.size()];
        final int rc = Native.viewApplyCut(handle, cut, oldToNew);
        if (rc == -4) {                                       // RAPID_EUUID_SEEN
            throw new MembershipView.UUIDAlreadySeenException(decidedCut.get(0), null);
        }
        if (rc != 0) {
            throw new IllegalStateException(Native.lastError());
        }
        final List<Endpoint> old = new ArrayList<>(byId);
        byId.clear();
        ids.clear();
        int n = 0;
        for (int oldId = 0; oldId < old.size(); oldId++) {
            if (oldToNew[oldId] >= 0) {
                n = Math.max(n, oldToNew[oldId] + 1);
            }
        }
        for (int i = 0; i < n; i++) {
            byId.add(null);
        }
        for (int oldId = 0; oldId < old.size(); oldId++) {
            final int q = oldToNew[oldId];
            if (q >= 0) {
                byId.set(q, old.get(oldId));
                ids.put(old.get(oldId), q);
            }
        }
        members = n;                                          // joiners that were not admitted are dropped
    }

    /** identifiersSeen on the device (MembershipView.java:58-60): NodeIds of the members, index = node id */
    void setNodeIds(final long[] idHigh, final long[] idLow) {
        if (Native.viewSetNodeIds(handle, idHigh, idLow) != 0) {
            throw new IllegalStateException(Native.lastError());
        }
    }

    /** getCurrentConfigurationId (:360-372) from the device-resident identifiersSeen and ring 0 */
    long getCurrentConfigurationId() {
        final long[] out = new long[1];
        if (Native.viewCurrentConfigId(handle, out) != 0) {
            throw new IllegalStateException(Native.lastError());
        }
        return out[0];
    }

    /**
     * Expansion of the monitoring overlay (rapid_view_overlay_spectrum): {lambda2, lambdaMin, residual, steps, lambda / 2K} of the
     * members' observer graph below its trivial eigenvalue 2K; lambda / 2K is the paper's expander figure.
     */
    double[] overlaySpectrum(final long seed, final double tol, final int maxSteps) {
        final long[] out = new long[5];
        if (Native.viewOverlaySpectrum(handle, seed, Double.doubleToRawLongBits(tol), maxSteps, out) != 0) {
            throw new IllegalStateException(Native.lastError());
        }
        final double lambda2 = Double.longBitsToDouble(out[0]);
        final double lambdaMin = Double.longBitsToDouble(out[1]);
        return new double[]{lambda2, lambdaMin, Double.longBitsToDouble(out[2]), out[3],
                            Math.max(Math.abs(lambda2), Math.abs(lambdaMin)) / (2.0 * K)};
    }

    /** id of a known endpoint (member or registered joiner), -1 otherwise; never registers anything */
    int tryIdOf(final Endpoint e) {
        final Integer id = ids.get(e);
        return id == null ? -1 : id;
    }

    int getMembershipSize() {                                 // :425-432
        return members;
    }

    List<Endpoint> getRing(final int k) {                     // :380-388
        final int[] out = new int[members];
        final int rc = Native.viewRing(handle, k, out);
        return map(out, rc < 0 ? rc : members);
    }

    List<Integer> getRingNumbers(final Endpoint observer, final Endpoint subject) {   // :397-418
        final int mask = Native.viewRingNumbers(handle, idOf(observer, false), idOf(subject, false));
        if (mask < 0) {
            throw new IllegalStateException(Native.lastError());
        }
        final List<Integer> rings = new ArrayList<>();
        for (int k = 0; k < K; k++) {
            if (((mask >> k) & 1) != 0) {
                rings.add(k);
            }
        }
        return rings;
    }

    /** :360-372, :544-556 — identifiersSeen is kept by the caller (NodeId high / low words, any order: sorted on the device) */
    long getCurrentConfigurationId(final long[] idHigh, final long[] idLow) {
        final long[] out = new long[1];
        if (Native.viewConfigId(handle, idHigh, idLow, out) != 0) {
            throw new IllegalStateException(Native.lastError());
        }
        return out[0];
    }

    List<Endpoint> getObserversOf(final Endpoint node) {      // :210-224
        return row(node, true);
    }

    List<Endpoint> getSubjectsOf(final Endpoint node) {       // :267-282
        return row(node, false);
    }

    List<Endpoint> getExpectedObserversOf(final Endpoint node) {   // :292-303
        final int[] out = new int[K];
        final int n = Native.viewExpectedObservers(handle, node.getHostname().toByteArray(), node.getPort(), out);
        return map(out, n);
    }

    private List<Endpoint> row(final Endpoint node, final boolean observers) {
        final Integer id = ids.get(node);
        if (id == null || id >= members) {
            throw new MembershipView.NodeNotInRingException(node);
        }
        final int[] out = new int[K];
        final int n = observers ? Native.viewObservers(handle, id, out) : Native.viewSubjects(handle, id, out);
        return map(out, n);
    }

    private List<Endpoint> map(final int[] out, final int n) {
        if (n < 0) {
            throw new IllegalStateException(Native.lastError());
        }
        final List<Endpoint> l = new ArrayList<>(n);
        for (int i = 0; i < n; i++) {
            l.add(byId.get(out[i]));
        }
        return l;
    }
}
