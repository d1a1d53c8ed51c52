"""H100-native stage-1 neural-atlas path: ctypes binding (`_native`), fused trainer (`atlas`),
synthetic inputs (`synth`)."""
