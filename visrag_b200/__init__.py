"""visrag_b200 — H100-native VisRAG-Ret embedding + retrieval hot path (hand-written sm_90a kernels
behind the reference's openmatch encode()/retrieve signatures). See DESIGN.md."""
__version__ = "0.1.0"
