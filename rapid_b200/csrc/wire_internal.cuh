// The decoded consensus messages of a rapid_wire handle, for the tallies that consume them on the device
// (classic_paxos.cu, fast_paxos.cu).  Only wire.cu knows the decoder's record layout and which kind was decoded last.
#pragma once

#include "common.cuh"

namespace rapid {

// Device arrays of the last consensus decode, in message order (valid until the next decode on the handle).  The classic-Paxos
// tallies also stage batches of host arrays in this shape; there cfg == NULL means the tallying handle's configuration and
// h2 == NULL means 0 for every message.
struct WireMsgs {
    int device;
    int64_t n;
    const int32_t* sender;              // id, -1 for an endpoint outside the dictionary
    const int64_t* cfg;
    const int32_t* rnd_round;           // rank (Phase1a) / rnd; 0 for FastRoundPhase2b
    const int32_t* rnd_node;
    const int32_t* vrnd_round;          // vrnd (Phase1b); 0 otherwise
    const int32_t* vrnd_node;
    const uint64_t* h1;                 // list fingerprint (rapid_proposal_fingerprint when every endpoint is known) + length
    const uint64_t* h2;
    const int32_t* len;
};

// RAPID_EINVAL (with the error set) unless the last decode on w was a successful consensus decode of `kind`.
int32_t wire_consensus_dev(const rapid_wire* w, int32_t kind, WireMsgs* out);

// The encoder's state of a rapid_wire handle (wire_encode.cu).  It has buffers of its own, so an encode never disturbs the last
// decode on the same handle, nor a decode the last encode.
struct WireEnc;
struct WireEncCtx {
    const View* view;
    int device;
    cudaStream_t stream;
    WireEnc** enc;                      // created by the first encode, freed with the handle
};
void wire_enc_ctx(rapid_wire* w, WireEncCtx* out);    // wire.cu
void wire_enc_free(WireEnc* e);                       // wire_encode.cu

// The alerts of a rapid_fdet's last interval (tick, then merge), for the encoder: alert i is (obs[i], subj[i], ring mask[i]);
// its first cell, cell_begin(i) = sum of popc(mask[j]) for j < i, carries its edgeStatus and configurationId.
struct FdetInterval {
    const View* view;
    int device;
    bool have;                          // a tick ran since the last reset, on the view as it still is
    int64_t n_alerts;
    const int32_t* obs;
    const int32_t* subj;
    const uint16_t* mask;
    const uint8_t* cell_status;
    const int64_t* cell_cfg;
};
void fdet_interval_dev(const rapid_fdet* fd, FdetInterval* out);   // fd.cu

// (round, node_index) -> one signed 64-bit word whose order is compareRanks' (Paxos.java:333-339)
RAPID_HD int64_t pack_rank(int32_t round, int32_t node) {
    return (int64_t)(((uint64_t)(uint32_t)round << 32) | (uint64_t)((uint32_t)node ^ 0x80000000u));
}
RAPID_HD int32_t rank_round(int64_t p) { return (int32_t)((uint64_t)p >> 32); }
RAPID_HD int32_t rank_node(int64_t p) { return (int32_t)((uint32_t)(uint64_t)p ^ 0x80000000u); }

// The answers of a rapid_pxa's last Phase1a (kind 1: Phase1b) or Phase2a (kind 2: Phase2b), for the encoder: answer i comes from
// acceptor sender[i] (acceptor_begin + local index) in ascending order; Phase1b answers carry vrnd[i] and the vval (h1, h2, len)[i],
// Phase2b answers all carry the Phase2a's value (v_h1, v_h2, v_len).  Ranks are packed as classic_paxos.cu packs them.
struct PxaAnswers {
    int device;
    int kind;                           // 0: no answers pending
    int64_t cfg, R, begin, n, rank;
    const int32_t* sender;
    const int64_t* vrnd;
    const uint64_t* h1;
    const uint64_t* h2;
    const int32_t* len;
    uint64_t v_h1, v_h2;
    int32_t v_len;
};
void pxa_answers_dev(const rapid_pxa* a, PxaAnswers* out);        // classic_paxos.cu

}  // namespace rapid
