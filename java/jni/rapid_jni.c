/*
 * JNI glue between com.vrg.rapid.gpu.Native and librapid_b200.so (include/rapid_b200.h).
 *
 * NOT compiled in this repository's build image: there is no JDK (no jni.h).  Where one exists:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../include rapid_jni.c \
 *       -L../../rapid_b200 -lrapid_b200 -o librapid_jni.so
 * Every native is a thin pass-through: pin / copy the Java arrays, call the C entry point, release.  Handles travel
 * as jlong.  No JNI exception is raised here: the Java side checks the status code and asks lastError().
 */
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "rapid_b200.h"

#define H(type, h) ((type*)(intptr_t)(h))
#define BUF(env, b) ((b) ? (*(env))->GetDirectBufferAddress((env), (b)) : NULL)

JNIEXPORT jstring JNICALL Java_com_vrg_rapid_gpu_Native_lastError(JNIEnv* env, jclass c) {
    char buf[512];
    rapid_last_error(buf, sizeof(buf));
    return (*env)->NewStringUTF(env, buf);
}

/* ---------------------------------------------------------------- MembershipView */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_viewCreate(JNIEnv* env, jclass c, jint k, jlong n, jbyteArray hostBytes,
                                                                 jintArray hostOff, jintArray port, jint device) {
    jbyte* hb = (*env)->GetByteArrayElements(env, hostBytes, NULL);
    jint* ho = (*env)->GetIntArrayElements(env, hostOff, NULL);
    jint* po = (*env)->GetIntArrayElements(env, port, NULL);
    rapid_view* v = NULL;
    const int32_t rc = rapid_view_create(&v, k, n, (const uint8_t*)hb, (const int32_t*)ho, (const int32_t*)po, device);
    (*env)->ReleaseByteArrayElements(env, hostBytes, hb, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, hostOff, ho, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, port, po, JNI_ABORT);
    return rc == RAPID_OK ? (jlong)(intptr_t)v : 0;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewDestroy(JNIEnv* env, jclass c, jlong view) {
    return rapid_view_destroy(H(rapid_view, view));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewRing(JNIEnv* env, jclass c, jlong view, jint ring, jintArray out) {
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    const int32_t rc = rapid_view_ring(H(rapid_view, view), ring, (int32_t*)o);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc;
}

static jint row_call(JNIEnv* env, jlong view, jint node, jintArray out, int observers) {
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    int32_t cnt = 0;
    const int32_t rc = observers ? rapid_view_observers(H(rapid_view, view), node, (int32_t*)o, &cnt)
                                 : rapid_view_subjects(H(rapid_view, view), node, (int32_t*)o, &cnt);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc == RAPID_OK ? cnt : rc;        /* RAPID_ENOT_IN_RING -> NodeNotInRingException on the Java side */
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewObservers(JNIEnv* env, jclass c, jlong view, jint node, jintArray out) {
    return row_call(env, view, node, out, 1);
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewSubjects(JNIEnv* env, jclass c, jlong view, jint node, jintArray out) {
    return row_call(env, view, node, out, 0);
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewExpectedObservers(JNIEnv* env, jclass c, jlong view, jbyteArray host,
                                                                           jint port, jintArray out) {
    const jsize len = (*env)->GetArrayLength(env, host);
    jbyte* h = (*env)->GetByteArrayElements(env, host, NULL);
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    int32_t cnt = 0;
    const int32_t rc = rapid_view_expected_observers(H(rapid_view, view), (const uint8_t*)h, len, port, (int32_t*)o, &cnt);
    (*env)->ReleaseByteArrayElements(env, host, h, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc == RAPID_OK ? cnt : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewRingNumbers(JNIEnv* env, jclass c, jlong view, jint observer, jint subject) {
    uint16_t m = 0;
    const int32_t rc = rapid_view_ring_numbers(H(rapid_view, view), observer, subject, &m);
    return rc == RAPID_OK ? (jint)m : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewConfigId(JNIEnv* env, jclass c, jlong view, jlongArray hi, jlongArray lo,
                                                                  jlongArray out1) {
    const jsize n = (*env)->GetArrayLength(env, hi);
    jlong* h = (*env)->GetLongArrayElements(env, hi, NULL);
    jlong* l = (*env)->GetLongArrayElements(env, lo, NULL);
    int64_t id = 0;
    const int32_t rc = rapid_view_config_id(H(rapid_view, view), (const int64_t*)h, (const int64_t*)l, n, &id);
    (*env)->ReleaseLongArrayElements(env, hi, h, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, lo, l, JNI_ABORT);
    const jlong v = id;
    (*env)->SetLongArrayRegion(env, out1, 0, 1, &v);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewRegisterJoiners(JNIEnv* env, jclass c, jlong view, jbyteArray hostBytes,
                                                                         jintArray hostOff, jintArray port) {
    const jsize n = (*env)->GetArrayLength(env, port);
    jbyte* hb = (*env)->GetByteArrayElements(env, hostBytes, NULL);
    jint* ho = (*env)->GetIntArrayElements(env, hostOff, NULL);
    jint* po = (*env)->GetIntArrayElements(env, port, NULL);
    int32_t first = 0;
    const int32_t rc = rapid_view_register_joiners(H(rapid_view, view), n, (const uint8_t*)hb, (const int32_t*)ho,
                                                   (const int32_t*)po, &first);
    (*env)->ReleaseByteArrayElements(env, hostBytes, hb, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, hostOff, ho, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, port, po, JNI_ABORT);
    return rc == RAPID_OK ? first : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewApplyCut(JNIEnv* env, jclass c, jlong view, jintArray cutIds, jintArray outOldToNew) {
    const jsize n = (*env)->GetArrayLength(env, cutIds);
    jint* ids = (*env)->GetIntArrayElements(env, cutIds, NULL);
    jint* map = outOldToNew ? (*env)->GetIntArrayElements(env, outOldToNew, NULL) : NULL;
    const int32_t rc = rapid_view_apply_cut(H(rapid_view, view), (const int32_t*)ids, n, (int32_t*)map);
    (*env)->ReleaseIntArrayElements(env, cutIds, ids, JNI_ABORT);
    if (map) (*env)->ReleaseIntArrayElements(env, outOldToNew, map, 0);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewSetNodeIds(JNIEnv* env, jclass c, jlong view, jlongArray idHigh, jlongArray idLow) {
    jlong* hi = (*env)->GetLongArrayElements(env, idHigh, NULL);
    jlong* lo = (*env)->GetLongArrayElements(env, idLow, NULL);
    const int32_t rc = rapid_view_set_node_ids(H(rapid_view, view), (const int64_t*)hi, (const int64_t*)lo);
    (*env)->ReleaseLongArrayElements(env, idHigh, hi, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, idLow, lo, JNI_ABORT);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewSetJoinerIds(JNIEnv* env, jclass c, jlong view, jint firstJoinerId, jlongArray idHigh,
                                                                      jlongArray idLow) {
    const jsize n = (*env)->GetArrayLength(env, idHigh);
    jlong* hi = (*env)->GetLongArrayElements(env, idHigh, NULL);
    jlong* lo = (*env)->GetLongArrayElements(env, idLow, NULL);
    const int32_t rc = rapid_view_set_joiner_ids(H(rapid_view, view), firstJoinerId, n, (const int64_t*)hi, (const int64_t*)lo);
    (*env)->ReleaseLongArrayElements(env, idHigh, hi, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, idLow, lo, JNI_ABORT);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewCurrentConfigId(JNIEnv* env, jclass c, jlong view, jlongArray out1) {
    int64_t v = 0;
    const int32_t rc = rapid_view_current_config_id(H(rapid_view, view), &v);
    const jlong j = (jlong)v;
    (*env)->SetLongArrayRegion(env, out1, 0, 1, &j);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_viewOverlaySpectrum(JNIEnv* env, jclass c, jlong view, jlong seed, jlong tolBits,
                                                                         jint maxSteps, jlongArray out5) {
    double tol, d[4] = {0.0, 0.0, 0.0, 0.0};
    int32_t steps = 0;
    float ms = 0.f;
    jlong out[5];
    memcpy(&tol, &tolBits, sizeof(tol));
    const int32_t rc = rapid_view_overlay_spectrum(H(rapid_view, view), (uint64_t)seed, tol, maxSteps, &d[0], &d[1], &d[2], &steps, &ms);
    d[3] = ms;
    memcpy(&out[0], &d[0], 3 * sizeof(double));
    out[3] = steps;
    memcpy(&out[4], &d[3], sizeof(double));
    if (rc == RAPID_OK) (*env)->SetLongArrayRegion(env, out5, 0, 5, out);
    return rc;
}

/* ---------------------------------------------------------------- cut detector */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_cdCreate(JNIEnv* env, jclass c, jlong view, jint h, jint l, jlong receivers,
                                                               jlong begin, jint flags, jlong maxSubjects) {
    rapid_cd* cd = NULL;
    const int32_t rc = rapid_cd_create(&cd, H(rapid_view, view), h, l, receivers, begin, (uint32_t)flags, maxSubjects);
    return rc == RAPID_OK ? (jlong)(intptr_t)cd : 0;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdDestroy(JNIEnv* env, jclass c, jlong cd) {
    return rapid_cd_destroy(H(rapid_cd, cd));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdApplyBatch(JNIEnv* env, jclass c, jlong cd, jlong cfg, jlong n, jobject dst,
                                                                  jobject ring, jobject status, jobject cellCfg, jint dflags,
                                                                  jobject blocked, jobject bitmap, jlong permSeed, jobject oh,
                                                                  jobject oh2, jobject olen, jobject oann) {
    rapid_delivery d;
    d.flags = (uint32_t)dflags;
    d.blocked = (const uint8_t*)BUF(env, blocked);
    d.bitmap = (const uint32_t*)BUF(env, bitmap);
    d.perm_seed = (uint64_t)permSeed;
    return rapid_cd_apply_batch(H(rapid_cd, cd), cfg, n, NULL, (const int32_t*)BUF(env, dst), (const uint8_t*)BUF(env, ring),
                                (const uint8_t*)BUF(env, status), (const int64_t*)BUF(env, cellCfg), dflags ? &d : NULL,
                                (uint64_t*)BUF(env, oh), (uint64_t*)BUF(env, oh2), (int32_t*)BUF(env, olen), (uint8_t*)BUF(env, oann));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdGetProposal(JNIEnv* env, jclass c, jlong cd, jlong receiver, jintArray out) {
    const jsize cap = (*env)->GetArrayLength(env, out);
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    int32_t len = 0;
    const int32_t rc = rapid_cd_get_proposal(H(rapid_cd, cd), receiver, (int32_t*)o, cap, &len);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc == RAPID_OK ? len : rc;
}

/* cutIds == NULL: no cut (in_cut reads -1); out2 = {n_classes, n_entries} */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdProposalCensus(JNIEnv* env, jclass c, jlong cd, jintArray cutIds, jlongArray out2) {
    const jsize n = cutIds ? (*env)->GetArrayLength(env, cutIds) : 0;
    jint* ids = cutIds ? (*env)->GetIntArrayElements(env, cutIds, NULL) : NULL;
    int64_t counts[2] = {0, 0};
    const int32_t rc = rapid_cd_proposal_census(H(rapid_cd, cd), (const int32_t*)ids, n, &counts[0], &counts[1]);
    if (ids) (*env)->ReleaseIntArrayElements(env, cutIds, ids, JNI_ABORT);
    if (rc == RAPID_OK) (*env)->SetLongArrayRegion(env, out2, 0, 2, (const jlong*)counts);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdReadCensus(JNIEnv* env, jclass c, jlong cd, jobject hash, jobject hash2, jobject len,
                                                                  jobject voters, jobject representative, jobject inCut, jobject listOff,
                                                                  jobject ids, jobject status) {
    return rapid_cd_read_census(H(rapid_cd, cd), (uint64_t*)BUF(env, hash), (uint64_t*)BUF(env, hash2), (int32_t*)BUF(env, len),
                                (int32_t*)BUF(env, voters), (int32_t*)BUF(env, representative), (int32_t*)BUF(env, inCut),
                                (int64_t*)BUF(env, listOff), (int32_t*)BUF(env, ids), (uint8_t*)BUF(env, status));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdReadCensusClasses(JNIEnv* env, jclass c, jlong cd, jintArray cls) {
    jint* o = (*env)->GetIntArrayElements(env, cls, NULL);
    const int32_t rc = rapid_cd_read_census_classes(H(rapid_cd, cd), (int32_t*)o);
    (*env)->ReleaseIntArrayElements(env, cls, o, 0);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdAggregate(JNIEnv* env, jclass c, jlong cd, jintArray dst, jbyteArray ring,
                                                                 jbyteArray status, jlong receiver, jintArray out) {
    const jsize n = (*env)->GetArrayLength(env, dst), cap = (*env)->GetArrayLength(env, out);
    jint* d = (*env)->GetIntArrayElements(env, dst, NULL);
    jbyte* r = (*env)->GetByteArrayElements(env, ring, NULL);
    jbyte* s = (*env)->GetByteArrayElements(env, status, NULL);
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    int32_t len = 0;
    const int32_t rc = rapid_cd_aggregate(H(rapid_cd, cd), n, NULL, (const int32_t*)d, (const uint8_t*)r, (const uint8_t*)s,
                                          receiver, (int32_t*)o, cap, &len);
    (*env)->ReleaseIntArrayElements(env, dst, d, JNI_ABORT);
    (*env)->ReleaseByteArrayElements(env, ring, r, JNI_ABORT);
    (*env)->ReleaseByteArrayElements(env, status, s, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc == RAPID_OK ? len : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdInvalidate(JNIEnv* env, jclass c, jlong cd, jlong receiver, jintArray out) {
    const jsize cap = (*env)->GetArrayLength(env, out);
    jint* o = (*env)->GetIntArrayElements(env, out, NULL);
    int32_t len = 0;
    const int32_t rc = rapid_cd_invalidate(H(rapid_cd, cd), receiver, (int32_t*)o, cap, &len);
    (*env)->ReleaseIntArrayElements(env, out, o, 0);
    return rc == RAPID_OK ? len : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdNumProposals(JNIEnv* env, jclass c, jlong cd, jlong receiver) {
    int32_t n = 0;
    const int32_t rc = rapid_cd_num_proposals(H(rapid_cd, cd), receiver, &n);
    return rc == RAPID_OK ? n : rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdClear(JNIEnv* env, jclass c, jlong cd) {
    return rapid_cd_clear(H(rapid_cd, cd));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdSequenceStats(JNIEnv* env, jclass c, jlong cd, jintArray out4) {
    int32_t v[4] = {0, 0, 0, 0};
    const int32_t rc = rapid_cd_sequence_stats(H(rapid_cd, cd), &v[0], &v[1], &v[2], &v[3]);
    jint* o = (*env)->GetIntArrayElements(env, out4, NULL);
    for (int i = 0; i < 4; ++i) o[i] = v[i];
    (*env)->ReleaseIntArrayElements(env, out4, o, 0);
    return rc;
}

/* ---------------------------------------------------------------- FastPaxos fast round */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_fpCreate(JNIEnv* env, jclass c, jlong cfg, jlong size, jlong cap, jint device) {
    rapid_fp* fp = NULL;
    const int32_t rc = rapid_fp_create(&fp, cfg, size, cap, device);
    return rc == RAPID_OK ? (jlong)(intptr_t)fp : 0;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpDestroy(JNIEnv* env, jclass c, jlong fp) {
    return rapid_fp_destroy(H(rapid_fp, fp));
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpReset(JNIEnv* env, jclass c, jlong fp, jlong cfg, jlong size) {
    return rapid_fp_reset(H(rapid_fp, fp), cfg, size);
}

static void put_result(JNIEnv* env, jlongArray out6, int32_t decided, uint64_t h1, uint64_t h2, int32_t len, int32_t count, int32_t recv) {
    const jlong v[6] = {decided, (jlong)h1, (jlong)h2, len, count, recv};
    (*env)->SetLongArrayRegion(env, out6, 0, 6, v);
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpTally(JNIEnv* env, jclass c, jlong fp, jintArray sender, jlongArray voteCfg,
                                                             jlongArray hash, jlongArray hash2, jintArray len, jlongArray out6) {
    const jsize n = (*env)->GetArrayLength(env, sender);
    jint* s = (*env)->GetIntArrayElements(env, sender, NULL);
    jlong* vc = voteCfg ? (*env)->GetLongArrayElements(env, voteCfg, NULL) : NULL;
    jlong* h1 = (*env)->GetLongArrayElements(env, hash, NULL);
    jlong* h2 = hash2 ? (*env)->GetLongArrayElements(env, hash2, NULL) : NULL;
    jint* ln = len ? (*env)->GetIntArrayElements(env, len, NULL) : NULL;
    int32_t decided = 0, dlen = 0, dcount = 0, recv = 0;
    uint64_t a = 0, b = 0;
    const int32_t rc = rapid_fp_tally(H(rapid_fp, fp), n, (const int32_t*)s, (const int64_t*)vc, (const uint64_t*)h1,
                                      (const uint64_t*)h2, (const int32_t*)ln, &decided, &a, &b, &dlen, &dcount, &recv);
    (*env)->ReleaseIntArrayElements(env, sender, s, JNI_ABORT);
    if (vc) (*env)->ReleaseLongArrayElements(env, voteCfg, vc, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, hash, h1, JNI_ABORT);
    if (h2) (*env)->ReleaseLongArrayElements(env, hash2, h2, JNI_ABORT);
    if (ln) (*env)->ReleaseIntArrayElements(env, len, ln, JNI_ABORT);
    put_result(env, out6, decided, a, b, dlen, dcount, recv);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpTallyCd(JNIEnv* env, jclass c, jlong fp, jlong cd, jlong comm, jlongArray out6) {
    int32_t decided = 0, dlen = 0, dcount = 0, recv = 0;
    uint64_t a = 0, b = 0;
    const int32_t rc = rapid_fp_tally_cd(H(rapid_fp, fp), H(rapid_cd, cd), H(rapid_comm, comm), &decided, &a, &b, &dlen, &dcount, &recv);
    put_result(env, out6, decided, a, b, dlen, dcount, recv);
    return rc;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpTallyCdAsync(JNIEnv* env, jclass c, jlong fp, jlong cd, jlong comm) {
    return rapid_fp_tally_cd_async(H(rapid_fp, fp), H(rapid_cd, cd), H(rapid_comm, comm));
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpResult(JNIEnv* env, jclass c, jlong fp, jlongArray out7) {
    int32_t decided = 0, dlen = 0, dcount = 0, recv = 0, in_call = -1;
    uint64_t a = 0, b = 0;
    const int32_t rc = rapid_fp_result(H(rapid_fp, fp), &decided, &a, &b, &dlen, &dcount, &recv, &in_call);
    put_result(env, out7, decided, a, b, dlen, dcount, recv);
    const jlong v = in_call;
    (*env)->SetLongArrayRegion(env, out7, 6, 1, &v);
    return rc;
}

JNIEXPORT jlongArray JNICALL Java_com_vrg_rapid_gpu_Native_proposalFingerprint(JNIEnv* env, jclass c, jintArray ids) {
    const jsize n = (*env)->GetArrayLength(env, ids);
    jint* p = (*env)->GetIntArrayElements(env, ids, NULL);
    uint64_t h1 = 0, h2 = 0;
    rapid_proposal_fingerprint((const int32_t*)p, n, &h1, &h2);
    (*env)->ReleaseIntArrayElements(env, ids, p, JNI_ABORT);
    jlongArray out = (*env)->NewLongArray(env, 2);
    const jlong v[2] = {(jlong)h1, (jlong)h2};
    (*env)->SetLongArrayRegion(env, out, 0, 2, v);
    return out;
}

/* ---------------------------------------------------------------- classic Paxos fallback (Paxos.java) */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_pxCreate(JNIEnv* env, jclass c, jlong cfg, jlong size, jlong cap, jint device) {
    rapid_px* px = NULL;
    const int32_t rc = rapid_px_create(&px, cfg, size, cap, device);
    return rc == RAPID_OK ? (jlong)(intptr_t)px : 0;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxDestroy(JNIEnv* env, jclass c, jlong px) { return rapid_px_destroy(H(rapid_px, px)); }

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxStartPhase1a(JNIEnv* env, jclass c, jlong px, jint round, jint nodeIndex) {
    int32_t started = 0;
    const int32_t rc = rapid_px_start_phase1a(H(rapid_px, px), round, nodeIndex, &started);
    return rc == RAPID_OK ? started : rc;
}

/* Paxos.selectProposalUsingCoordinatorRule (Paxos.java:271-328) */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_pxCoordinatorRule(JNIEnv* env, jclass c, jlong px, jintArray vrRound, jintArray vrNode,
                                                                        jlongArray hash, jlongArray hash2, jintArray len) {
    const jsize n = (*env)->GetArrayLength(env, len);
    jint* r0 = (*env)->GetIntArrayElements(env, vrRound, NULL);
    jint* r1 = (*env)->GetIntArrayElements(env, vrNode, NULL);
    jlong* h1 = (*env)->GetLongArrayElements(env, hash, NULL);
    jlong* h2 = hash2 ? (*env)->GetLongArrayElements(env, hash2, NULL) : NULL;
    jint* ln = (*env)->GetIntArrayElements(env, len, NULL);
    int64_t chosen = -1;
    const int32_t rc = rapid_px_coordinator_rule(H(rapid_px, px), n, (const int32_t*)r0, (const int32_t*)r1, (const uint64_t*)h1,
                                                 (const uint64_t*)h2, (const int32_t*)ln, &chosen);
    (*env)->ReleaseIntArrayElements(env, vrRound, r0, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, vrNode, r1, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, hash, h1, JNI_ABORT);
    if (h2) (*env)->ReleaseLongArrayElements(env, hash2, h2, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, len, ln, JNI_ABORT);
    return rc == RAPID_OK ? (jlong)chosen : (jlong)rc - 2;
}

/* Paxos.handlePhase1bMessage (Paxos.java:159-191) for a batch */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase1b(JNIEnv* env, jclass c, jlong px, jlongArray msgCfg, jintArray rndRound,
                                                               jintArray rndNode, jintArray vrRound, jintArray vrNode, jlongArray hash,
                                                               jlongArray hash2, jintArray len, jlongArray out6) {
    const jsize n = (*env)->GetArrayLength(env, len);
    jlong* mc = msgCfg ? (*env)->GetLongArrayElements(env, msgCfg, NULL) : NULL;
    jint* a0 = (*env)->GetIntArrayElements(env, rndRound, NULL);
    jint* a1 = (*env)->GetIntArrayElements(env, rndNode, NULL);
    jint* b0 = (*env)->GetIntArrayElements(env, vrRound, NULL);
    jint* b1 = (*env)->GetIntArrayElements(env, vrNode, NULL);
    jlong* h1 = (*env)->GetLongArrayElements(env, hash, NULL);
    jlong* h2 = hash2 ? (*env)->GetLongArrayElements(env, hash2, NULL) : NULL;
    jint* ln = (*env)->GetIntArrayElements(env, len, NULL);
    int32_t proposed = 0, clen = 0;
    int64_t trigger = -1, total = 0;
    uint64_t ca = 0, cb = 0;
    const int32_t rc = rapid_px_phase1b(H(rapid_px, px), n, (const int64_t*)mc, (const int32_t*)a0, (const int32_t*)a1, (const int32_t*)b0,
                                        (const int32_t*)b1, (const uint64_t*)h1, (const uint64_t*)h2, (const int32_t*)ln, &proposed,
                                        &trigger, &ca, &cb, &clen, &total);
    if (mc) (*env)->ReleaseLongArrayElements(env, msgCfg, mc, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, rndRound, a0, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, rndNode, a1, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, vrRound, b0, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, vrNode, b1, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, hash, h1, JNI_ABORT);
    if (h2) (*env)->ReleaseLongArrayElements(env, hash2, h2, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, len, ln, JNI_ABORT);
    const jlong v[6] = {proposed, (jlong)trigger, (jlong)ca, (jlong)cb, clen, (jlong)total};
    (*env)->SetLongArrayRegion(env, out6, 0, 6, v);
    return rc;
}

/* Paxos.handlePhase2bMessage (Paxos.java:223-236) for a batch */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase2b(JNIEnv* env, jclass c, jlong px, jlongArray msgCfg, jintArray rndRound,
                                                               jintArray rndNode, jintArray sender, jlongArray hash, jlongArray hash2,
                                                               jintArray len, jlongArray out5) {
    const jsize n = (*env)->GetArrayLength(env, len);
    jlong* mc = msgCfg ? (*env)->GetLongArrayElements(env, msgCfg, NULL) : NULL;
    jint* a0 = (*env)->GetIntArrayElements(env, rndRound, NULL);
    jint* a1 = (*env)->GetIntArrayElements(env, rndNode, NULL);
    jint* s = (*env)->GetIntArrayElements(env, sender, NULL);
    jlong* h1 = (*env)->GetLongArrayElements(env, hash, NULL);
    jlong* h2 = hash2 ? (*env)->GetLongArrayElements(env, hash2, NULL) : NULL;
    jint* ln = (*env)->GetIntArrayElements(env, len, NULL);
    int32_t decided = 0, dlen = 0;
    int64_t at = -1;
    uint64_t da = 0, db = 0;
    const int32_t rc = rapid_px_phase2b(H(rapid_px, px), n, (const int64_t*)mc, (const int32_t*)a0, (const int32_t*)a1, (const int32_t*)s,
                                        (const uint64_t*)h1, (const uint64_t*)h2, (const int32_t*)ln, &decided, &at, &da, &db, &dlen);
    if (mc) (*env)->ReleaseLongArrayElements(env, msgCfg, mc, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, rndRound, a0, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, rndNode, a1, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, sender, s, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, hash, h1, JNI_ABORT);
    if (h2) (*env)->ReleaseLongArrayElements(env, hash2, h2, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, len, ln, JNI_ABORT);
    const jlong v[5] = {decided, (jlong)at, (jlong)da, (jlong)db, dlen};
    (*env)->SetLongArrayRegion(env, out5, 0, 5, v);
    return rc;
}

JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_pxaCreate(JNIEnv* env, jclass c, jlong cfg, jlong n, jlong begin, jint device) {
    rapid_pxa* a = NULL;
    const int32_t rc = rapid_pxa_create(&a, cfg, n, begin, device);
    return rc == RAPID_OK ? (jlong)(intptr_t)a : 0;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxaDestroy(JNIEnv* env, jclass c, jlong a) { return rapid_pxa_destroy(H(rapid_pxa, a)); }
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxaRegisterFastRoundVotesCd(JNIEnv* env, jclass c, jlong a, jlong cd) {
    return rapid_pxa_register_fast_round_votes_cd(H(rapid_pxa, a), H(rapid_cd, cd));
}
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_pxaPhase1a(JNIEnv* env, jclass c, jlong a, jlong cfg, jint round, jint node) {
    int64_t n = 0;
    const int32_t rc = rapid_pxa_phase1a(H(rapid_pxa, a), cfg, round, node, &n);
    return rc == RAPID_OK ? (jlong)n : (jlong)rc;
}
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_pxaPhase2a(JNIEnv* env, jclass c, jlong a, jlong cfg, jint round, jint node, jlong h1,
                                                                 jlong h2, jint len) {
    int64_t n = 0;
    const int32_t rc = rapid_pxa_phase2a(H(rapid_pxa, a), cfg, round, node, (uint64_t)h1, (uint64_t)h2, len, &n);
    return rc == RAPID_OK ? (jlong)n : (jlong)rc;
}
/* jlong[] of handles -> rapid_pxa* array (malloc'ed; NULL if out of memory, which the entry point refuses as a NULL list) */
static const rapid_pxa** shard_list(JNIEnv* env, jlongArray shards, jint* n) {
    *n = (*env)->GetArrayLength(env, shards);
    const rapid_pxa** out = (const rapid_pxa**)malloc(sizeof(rapid_pxa*) * (size_t)(*n > 0 ? *n : 1));
    jlong* h = (*env)->GetLongArrayElements(env, shards, NULL);
    for (jint i = 0; out && i < *n; ++i) out[i] = H(rapid_pxa, h[i]);
    (*env)->ReleaseLongArrayElements(env, shards, h, JNI_ABORT);
    return out;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase1bFromAcceptorShards(JNIEnv* env, jclass c, jlong px, jlongArray shards, jlong comm,
                                                                                  jlong seed, jlongArray out6) {
    int32_t proposed = 0, clen = 0;
    int64_t trigger = -1, total = 0;
    uint64_t ca = 0, cb = 0;
    jint n = 0;
    const rapid_pxa** list = shard_list(env, shards, &n);
    const int32_t rc = rapid_px_phase1b_from_acceptor_shards(H(rapid_px, px), list, n, H(rapid_comm, comm), (uint64_t)seed, &proposed,
                                                             &trigger, &ca, &cb, &clen, &total);
    free(list);
    const jlong v[6] = {proposed, (jlong)trigger, (jlong)ca, (jlong)cb, clen, (jlong)total};
    (*env)->SetLongArrayRegion(env, out6, 0, 6, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase2bFromAcceptorShards(JNIEnv* env, jclass c, jlong px, jlongArray shards, jlong comm,
                                                                                  jlong seed, jlongArray out5) {
    int32_t decided = 0, dlen = 0;
    int64_t at = -1;
    uint64_t da = 0, db = 0;
    jint n = 0;
    const rapid_pxa** list = shard_list(env, shards, &n);
    const int32_t rc = rapid_px_phase2b_from_acceptor_shards(H(rapid_px, px), list, n, H(rapid_comm, comm), (uint64_t)seed, &decided, &at,
                                                             &da, &db, &dlen);
    free(list);
    const jlong v[5] = {decided, (jlong)at, (jlong)da, (jlong)db, dlen};
    (*env)->SetLongArrayRegion(env, out5, 0, 5, v);
    return rc;
}

/* ---------------------------------------------------------------- wire-format ingest (rapid.proto) */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_wireCreate(JNIEnv* env, jclass c, jlong view) {
    rapid_wire* w = NULL;
    const int32_t rc = rapid_wire_create(&w, H(rapid_view, view));
    return rc == RAPID_OK ? (jlong)(intptr_t)w : 0;
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireSetConfiguration(JNIEnv* env, jclass c, jlong wire, jlong cfgId) {
    return rapid_wire_set_configuration(H(rapid_wire, wire), cfgId);
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireDestroy(JNIEnv* env, jclass c, jlong w) { return rapid_wire_destroy(H(rapid_wire, w)); }

/* what the gRPC server hands to MembershipService.handleMessage (MembershipService.java:174), still serialized */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireDecodeAlerts(JNIEnv* env, jclass c, jlong w, jobject bytes, jint len,
                                                                      jboolean asRequest, jlongArray out5) {
    int64_t nm = 0, nc = 0, nd = 0, nj = 0;
    int32_t sender = -1;
    const int32_t rc = rapid_wire_decode_alerts(H(rapid_wire, w), (const uint8_t*)BUF(env, bytes), len, asRequest ? RAPID_WIRE_REQUEST : 0,
                                                &nm, &nc, &nd, &nj, &sender);
    const jlong v[5] = {(jlong)nm, (jlong)nc, (jlong)nd, (jlong)nj, sender};
    (*env)->SetLongArrayRegion(env, out5, 0, 5, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireApplyToDetector(JNIEnv* env, jclass c, jlong w, jlong cd, jlong cfg, jlong nCells) {
    const int32_t *src, *dst;
    const uint8_t *ring, *status;
    const int64_t* cell_cfg;
    int32_t rc = rapid_wire_cells_dev(H(rapid_wire, w), &src, &dst, &ring, &status, &cell_cfg);
    if (rc != RAPID_OK) return rc;
    return rapid_cd_apply_batch_dev(H(rapid_cd, cd), cfg, nCells, src, dst, ring, status, cell_cfg, NULL);
}

JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireApplyToDetectorAsync(JNIEnv* env, jclass c, jlong w, jlong cd, jlong cfg, jlong nCells) {
    const int32_t *src, *dst;
    const uint8_t *ring, *status;
    const int64_t* cell_cfg;
    int32_t rc = rapid_wire_cells_dev(H(rapid_wire, w), &src, &dst, &ring, &status, &cell_cfg);
    if (rc != RAPID_OK) return rc;
    return rapid_cd_apply_batch_dev_async(H(rapid_cd, cd), cfg, nCells, src, dst, ring, status, cell_cfg, NULL);
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdSync(JNIEnv* env, jclass c, jlong cd) { return rapid_cd_sync(H(rapid_cd, cd)); }

/* consensus messages of one kind, as the host split a drained inbox by RapidRequest content case */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireDecodeConsensus(JNIEnv* env, jclass c, jlong w, jint kind, jobject bytes, jlongArray off,
                                                                         jboolean asRequest, jlongArray out2) {
    const jsize n = (*env)->GetArrayLength(env, off) - 1;
    jlong* o = (*env)->GetLongArrayElements(env, off, NULL);
    int64_t us = 0, ue = 0;
    const int32_t rc = rapid_wire_decode_consensus(H(rapid_wire, w), kind, (const uint8_t*)BUF(env, bytes), (const int64_t*)o, n < 0 ? 0 : n,
                                                   asRequest ? RAPID_WIRE_REQUEST : 0, &us, &ue);
    (*env)->ReleaseLongArrayElements(env, off, o, JNI_ABORT);
    const jlong v[2] = {(jlong)us, (jlong)ue};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodeAlertBatches(JNIEnv* env, jclass c, jlong w, jlong fd, jboolean asRequest,
                                                                            jlongArray out2) {
    int64_t n = 0, bytes = 0;
    const int32_t rc = rapid_wire_encode_alert_batches(H(rapid_wire, w), H(rapid_fdet, fd), asRequest ? RAPID_WIRE_REQUEST : 0, &n, &bytes);
    const jlong v[2] = {(jlong)n, (jlong)bytes};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodeVotes(JNIEnv* env, jclass c, jlong w, jlong cd, jlong cfg, jboolean asRequest,
                                                                     jlongArray out2) {
    int64_t n = 0, nb = 0;
    const int32_t rc = rapid_wire_encode_votes(H(rapid_wire, w), H(rapid_cd, cd), cfg, asRequest ? RAPID_WIRE_REQUEST : 0, &n, &nb);
    const jlong v[2] = {(jlong)n, (jlong)nb};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodedCounts(JNIEnv* env, jclass c, jlong w, jlongArray out4) {
    int64_t a = 0, b = 0, d = 0, e = 0;
    const int32_t rc = rapid_wire_encoded_counts(H(rapid_wire, w), &a, &b, &d, &e);
    const jlong v[4] = {(jlong)a, (jlong)b, (jlong)d, (jlong)e};
    (*env)->SetLongArrayRegion(env, out4, 0, 4, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodedDev(JNIEnv* env, jclass c, jlong w, jlongArray out5) {
    const uint8_t *hdr = NULL, *bodies = NULL;
    const int64_t *hoff = NULL, *boff = NULL;
    const int32_t* bid = NULL;
    const int32_t rc = rapid_wire_encoded_dev(H(rapid_wire, w), &hdr, &hoff, &bid, &bodies, &boff);
    const jlong v[5] = {(jlong)(intptr_t)hdr, (jlong)(intptr_t)hoff, (jlong)(intptr_t)bid, (jlong)(intptr_t)bodies, (jlong)(intptr_t)boff};
    (*env)->SetLongArrayRegion(env, out5, 0, 5, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodePhase1b(JNIEnv* env, jclass c, jlong w, jlong pxa, jlong cd, jboolean asRequest,
                                                                       jlongArray out2) {
    int64_t n = 0, nb = 0;
    const int32_t rc = rapid_wire_encode_phase1b(H(rapid_wire, w), H(rapid_pxa, pxa), H(rapid_cd, cd), asRequest ? RAPID_WIRE_REQUEST : 0, &n, &nb);
    const jlong v[2] = {(jlong)n, (jlong)nb};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireEncodePhase2b(JNIEnv* env, jclass c, jlong w, jlong pxa, jlong cd, jboolean asRequest,
                                                                       jlongArray out2) {
    int64_t n = 0, nb = 0;
    const int32_t rc = rapid_wire_encode_phase2b(H(rapid_wire, w), H(rapid_pxa, pxa), H(rapid_cd, cd), asRequest ? RAPID_WIRE_REQUEST : 0, &n, &nb);
    const jlong v[2] = {(jlong)n, (jlong)nb};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
/* the read-backs write counts of the last encode: a Java array shorter than that is refused before anything is written */
static int enc_short(JNIEnv* env, jarray a, int64_t need) { return a && (int64_t)(*env)->GetArrayLength(env, a) < need; }
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireReadEncoded(JNIEnv* env, jclass c, jlong w, jbyteArray headers, jlongArray headerOff,
                                                                     jintArray bodyId, jbyteArray bodies, jlongArray bodyOff) {
    int64_t n = 0, hb = 0, nb = 0, bb = 0;
    int32_t rc = rapid_wire_encoded_counts(H(rapid_wire, w), &n, &hb, &nb, &bb);
    if (rc) return rc;
    if (enc_short(env, headers, hb) || enc_short(env, headerOff, n + 1) || enc_short(env, bodyId, n) || enc_short(env, bodies, bb) ||
        enc_short(env, bodyOff, nb + 1)) return RAPID_EINVAL;
    jbyte* h = headers ? (*env)->GetByteArrayElements(env, headers, NULL) : NULL;
    jlong* ho = headerOff ? (*env)->GetLongArrayElements(env, headerOff, NULL) : NULL;
    jint* bi = bodyId ? (*env)->GetIntArrayElements(env, bodyId, NULL) : NULL;
    jbyte* b = bodies ? (*env)->GetByteArrayElements(env, bodies, NULL) : NULL;
    jlong* bo = bodyOff ? (*env)->GetLongArrayElements(env, bodyOff, NULL) : NULL;
    rc = rapid_wire_read_encoded(H(rapid_wire, w), (uint8_t*)h, (int64_t*)ho, (int32_t*)bi, (uint8_t*)b, (int64_t*)bo);
    if (h) (*env)->ReleaseByteArrayElements(env, headers, h, 0);
    if (ho) (*env)->ReleaseLongArrayElements(env, headerOff, ho, 0);
    if (bi) (*env)->ReleaseIntArrayElements(env, bodyId, bi, 0);
    if (b) (*env)->ReleaseByteArrayElements(env, bodies, b, 0);
    if (bo) (*env)->ReleaseLongArrayElements(env, bodyOff, bo, 0);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireReadEncodedSizes(JNIEnv* env, jclass c, jlong w, jlongArray sizes) {
    int64_t n = 0;
    int32_t rc = rapid_wire_encoded_counts(H(rapid_wire, w), &n, NULL, NULL, NULL);
    if (rc) return rc;
    if (!sizes || enc_short(env, sizes, n)) return RAPID_EINVAL;
    jlong* s = (*env)->GetLongArrayElements(env, sizes, NULL);
    rc = rapid_wire_read_encoded_sizes(H(rapid_wire, w), (int64_t*)s);
    (*env)->ReleaseLongArrayElements(env, sizes, s, 0);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireReadEncodedSenders(JNIEnv* env, jclass c, jlong w, jintArray sender) {
    int64_t n = 0;
    int32_t rc = rapid_wire_encoded_counts(H(rapid_wire, w), &n, NULL, NULL, NULL);
    if (rc) return rc;
    if (!sender || enc_short(env, sender, n)) return RAPID_EINVAL;
    jint* s = (*env)->GetIntArrayElements(env, sender, NULL);
    rc = rapid_wire_read_encoded_senders(H(rapid_wire, w), (int32_t*)s);
    (*env)->ReleaseIntArrayElements(env, sender, s, 0);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireReadConsensus(JNIEnv* env, jclass c, jlong w, jintArray sender, jlongArray cfg,
                                                                       jintArray rndRound, jintArray rndNode, jintArray vrndRound,
                                                                       jintArray vrndNode, jlongArray hash, jlongArray hash2, jintArray len) {
    jint* s = sender ? (*env)->GetIntArrayElements(env, sender, NULL) : NULL;
    jlong* cf = cfg ? (*env)->GetLongArrayElements(env, cfg, NULL) : NULL;
    jint* a0 = rndRound ? (*env)->GetIntArrayElements(env, rndRound, NULL) : NULL;
    jint* a1 = rndNode ? (*env)->GetIntArrayElements(env, rndNode, NULL) : NULL;
    jint* b0 = vrndRound ? (*env)->GetIntArrayElements(env, vrndRound, NULL) : NULL;
    jint* b1 = vrndNode ? (*env)->GetIntArrayElements(env, vrndNode, NULL) : NULL;
    jlong* h1 = hash ? (*env)->GetLongArrayElements(env, hash, NULL) : NULL;
    jlong* h2 = hash2 ? (*env)->GetLongArrayElements(env, hash2, NULL) : NULL;
    jint* ln = len ? (*env)->GetIntArrayElements(env, len, NULL) : NULL;
    const int32_t rc = rapid_wire_read_consensus(H(rapid_wire, w), (int32_t*)s, (int64_t*)cf, (int32_t*)a0, (int32_t*)a1, (int32_t*)b0,
                                                 (int32_t*)b1, (uint64_t*)h1, (uint64_t*)h2, (int32_t*)ln);
    if (s) (*env)->ReleaseIntArrayElements(env, sender, s, 0);
    if (cf) (*env)->ReleaseLongArrayElements(env, cfg, cf, 0);
    if (a0) (*env)->ReleaseIntArrayElements(env, rndRound, a0, 0);
    if (a1) (*env)->ReleaseIntArrayElements(env, rndNode, a1, 0);
    if (b0) (*env)->ReleaseIntArrayElements(env, vrndRound, b0, 0);
    if (b1) (*env)->ReleaseIntArrayElements(env, vrndNode, b1, 0);
    if (h1) (*env)->ReleaseLongArrayElements(env, hash, h1, 0);
    if (h2) (*env)->ReleaseLongArrayElements(env, hash2, h2, 0);
    if (ln) (*env)->ReleaseIntArrayElements(env, len, ln, 0);
    return rc;
}
/* the cval / decision list of a trigger_index / decided_index, without a protobuf runtime */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_wireConsensusValue(JNIEnv* env, jclass c, jlong w, jlong index, jintArray outIds) {
    const jsize cap = outIds ? (*env)->GetArrayLength(env, outIds) : 0;
    jint* o = outIds ? (*env)->GetIntArrayElements(env, outIds, NULL) : NULL;
    int32_t len = 0;
    const int32_t rc = rapid_wire_consensus_value(H(rapid_wire, w), index, (int32_t*)o, cap, &len);
    if (o) (*env)->ReleaseIntArrayElements(env, outIds, o, 0);
    return rc == RAPID_OK ? len : rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase1bWire(JNIEnv* env, jclass c, jlong px, jlong w, jlongArray out6) {
    int32_t proposed = 0, clen = 0;
    int64_t trigger = -1, total = 0;
    uint64_t ca = 0, cb = 0;
    const int32_t rc = rapid_px_phase1b_wire(H(rapid_px, px), H(rapid_wire, w), &proposed, &trigger, &ca, &cb, &clen, &total);
    const jlong v[6] = {proposed, (jlong)trigger, (jlong)ca, (jlong)cb, clen, (jlong)total};
    (*env)->SetLongArrayRegion(env, out6, 0, 6, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_pxPhase2bWire(JNIEnv* env, jclass c, jlong px, jlong w, jlongArray out5) {
    int32_t decided = 0, dlen = 0;
    int64_t at = -1;
    uint64_t da = 0, db = 0;
    const int32_t rc = rapid_px_phase2b_wire(H(rapid_px, px), H(rapid_wire, w), &decided, &at, &da, &db, &dlen);
    const jlong v[5] = {decided, (jlong)at, (jlong)da, (jlong)db, dlen};
    (*env)->SetLongArrayRegion(env, out5, 0, 5, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fpTallyWire(JNIEnv* env, jclass c, jlong fp, jlong w, jlongArray out6) {
    int32_t decided = 0, dlen = 0, dcount = 0, recv = 0;
    uint64_t a = 0, b = 0;
    const int32_t rc = rapid_fp_tally_wire(H(rapid_fp, fp), H(rapid_wire, w), &decided, &a, &b, &dlen, &dcount, &recv);
    put_result(env, out6, decided, a, b, dlen, dcount, recv);
    return rc;
}

/* ---------------------------------------------------------------- alert generation (PingPongFailureDetector.java) */
JNIEXPORT jlong JNICALL Java_com_vrg_rapid_gpu_Native_fdetCreate(JNIEnv* env, jclass c, jlong view, jint thr, jint bootThr) {
    rapid_fdet* fd = NULL;
    const int32_t rc = rapid_fdet_create(&fd, H(rapid_view, view), thr, bootThr);
    return rc == RAPID_OK ? (jlong)(intptr_t)fd : 0;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fdetDestroy(JNIEnv* env, jclass c, jlong fd) { return rapid_fdet_destroy(H(rapid_fdet, fd)); }
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fdetReset(JNIEnv* env, jclass c, jlong fd) { return rapid_fdet_reset(H(rapid_fdet, fd)); }

/* what the msbg thread's scheduleAtFixedRate of every detector amounts to (MembershipService.java:697-707), for all virtual nodes */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fdetTick(JNIEnv* env, jclass c, jlong fd, jbyteArray nodeFlags, jbyteArray edgeFail,
                                                              jlong cfg, jlongArray out2) {
    jbyte* nf = (*env)->GetByteArrayElements(env, nodeFlags, NULL);
    jbyte* ef = edgeFail ? (*env)->GetByteArrayElements(env, edgeFail, NULL) : NULL;
    int64_t na = 0, nc = 0;
    const int32_t rc = rapid_fdet_tick(H(rapid_fdet, fd), (const uint8_t*)nf, (const uint8_t*)ef, cfg, &na, &nc);
    (*env)->ReleaseByteArrayElements(env, nodeFlags, nf, JNI_ABORT);
    if (ef) (*env)->ReleaseByteArrayElements(env, edgeFail, ef, JNI_ABORT);
    const jlong v[2] = {(jlong)na, (jlong)nc};
    (*env)->SetLongArrayRegion(env, out2, 0, 2, v);
    return rc;
}
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_fdetApplyToDetector(JNIEnv* env, jclass c, jlong fd, jlong cd, jlong cfg, jlong nCells) {
    const int32_t *src, *dst;
    const uint8_t *ring, *status;
    const int64_t* cell_cfg;
    int32_t rc = rapid_fdet_cells_dev(H(rapid_fdet, fd), &src, &dst, &ring, &status, &cell_cfg);
    if (rc != RAPID_OK) return rc;
    return rapid_cd_apply_batch_dev(H(rapid_cd, cd), cfg, nCells, src, dst, ring, status, cell_cfg, NULL);
}

/* ---------------------------------------------------------------- a drained inbox of BatchedAlertMessages (MembershipService.java:300-354 per batch) */
JNIEXPORT jint JNICALL Java_com_vrg_rapid_gpu_Native_cdApplyBatches(JNIEnv* env, jclass c, jlong cd, jlong cfg, jintArray dst, jbyteArray ring,
                                                                    jbyteArray status, jlongArray cellCfg, jlongArray batchOff, jobject outHash,
                                                                    jobject outHash2, jobject outLen, jobject outAnnounced, jobject outAnnouncedIn) {
    const jsize n = (*env)->GetArrayLength(env, dst);
    const jsize nb = (*env)->GetArrayLength(env, batchOff) - 1;
    jint* d = (*env)->GetIntArrayElements(env, dst, NULL);
    jbyte* r = (*env)->GetByteArrayElements(env, ring, NULL);
    jbyte* s = (*env)->GetByteArrayElements(env, status, NULL);
    jlong* cc = cellCfg ? (*env)->GetLongArrayElements(env, cellCfg, NULL) : NULL;
    jlong* off = (*env)->GetLongArrayElements(env, batchOff, NULL);
    const int32_t rc = rapid_cd_apply_batches(H(rapid_cd, cd), cfg, n, NULL, (const int32_t*)d, (const uint8_t*)r, (const uint8_t*)s,
                                              (const int64_t*)cc, nb, (const int64_t*)off, NULL, (uint64_t*)BUF(env, outHash),
                                              (uint64_t*)BUF(env, outHash2), (int32_t*)BUF(env, outLen), (uint8_t*)BUF(env, outAnnounced),
                                              (int32_t*)BUF(env, outAnnouncedIn));
    (*env)->ReleaseIntArrayElements(env, dst, d, JNI_ABORT);
    (*env)->ReleaseByteArrayElements(env, ring, r, JNI_ABORT);
    (*env)->ReleaseByteArrayElements(env, status, s, JNI_ABORT);
    if (cc) (*env)->ReleaseLongArrayElements(env, cellCfg, cc, JNI_ABORT);
    (*env)->ReleaseLongArrayElements(env, batchOff, off, JNI_ABORT);
    return rc;
}
