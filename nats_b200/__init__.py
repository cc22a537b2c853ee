"""nats_b200 -- H100-native (sm_90a) implementation of the hot path of lukecq1231/nats.

    from nats_b200 import nats          # the reference-compatible module (scripts/nats.py surface)

The compute lives in libnats_b200.so (nats_b200/csrc, include/nats_b200.h); there is no CPU fallback."""
__all__ = ['nats', 'data_iterator']
