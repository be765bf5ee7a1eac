"""d3feat_b200 -- Hopper-native (sm_90a) implementation of the D3Feat dense feature-extraction hot path:
grid subsampling -> radius neighbours -> KPConv pyramid (KPFCNN encoder), behind the reference's operator
signatures. Host code is Python; all device code is hand-written CUDA behind the C ABI in
include/d3feat_b200.h (d3feat_b200/libd3feat_b200.so). There is no CPU fallback."""

__all__ = ["synth", "tf_custom_ops", "cpp_subsampling", "convolution_ops", "network_blocks", "pyramid", "encoder"]
