"""mertools_b200 — H100-native (sm_90a) implementation of the MERTools hot path: tri-modal feature extraction
(``mertools_b200.extract``) and Attention-fusion training (``mertools_b200.fusion``, ``mertools_b200.main_release``)
behind the reference's own function / script / .npy contract, over the C ABI of ``include/mer_b200.h``
(``lib/libmer_b200.so``, built by ``python -m mertools_b200._build``).  No CPU fallback: every entry point runs on
the device or raises."""

__version__ = "0.2.0"
