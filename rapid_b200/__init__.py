"""rapid_b200 — H100-native cut detection + fast-round tally for the Rapid membership protocol.

The product is rapid_b200/librapid_b200.so (hand-written sm_90a CUDA behind the C ABI of include/rapid_b200.h);
these modules mirror the reference's Java classes on top of it.  No CPU fallback exists.
"""
from . import _native
from ._native import (RapidError, NodeNotInRingException, NodeAlreadyInRingException, UUIDAlreadySeenException,
                      HashCollisionError)
from .membership_view import MembershipView
from .cut_detector import MultiNodeCutDetector, VirtualCluster, proposal_fingerprint, UP, DOWN
from .fast_paxos import FastPaxos, NcclComm, quorum
from .classic_paxos import Paxos, PaxosAcceptors
from .wire import EncodedMessages, WireDecoder
from .failure_detector import EdgeFailureDetectors
from .simulation import ClusterSimulation

__all__ = ["MembershipView", "MultiNodeCutDetector", "VirtualCluster", "FastPaxos", "NcclComm", "quorum", "Paxos", "PaxosAcceptors", "WireDecoder", "EncodedMessages", "EdgeFailureDetectors", "ClusterSimulation",
           "proposal_fingerprint", "UP", "DOWN", "RapidError", "NodeNotInRingException",
           "NodeAlreadyInRingException", "UUIDAlreadySeenException", "HashCollisionError"]
