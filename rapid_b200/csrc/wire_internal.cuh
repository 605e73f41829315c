// The decoded consensus messages of a rapid_wire handle, for the tallies that consume them on the device
// (classic_paxos.cu, fast_paxos.cu).  Only wire.cu knows the decoder's record layout and which kind was decoded last.
#pragma once

#include "common.cuh"

namespace rapid {

// Device arrays of the last consensus decode, in message order (valid until the next decode on the handle).
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

}  // namespace rapid
