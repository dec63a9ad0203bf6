"""kaito_b200 -- H100-native retrieval engine behind KAITO's RAGService /retrieve and /index.

`kaito_b200._native` binds libkaito_rag.so (hand-written sm_90a CUDA, C ABI in
include/kaito_rag.h).  The host-side mirror of the reference's RAGService classes lives in
`kaito_b200.vector_store` / `kaito_b200.retriever`.  There is no CPU fallback.
"""
__version__ = "0.1.0"
