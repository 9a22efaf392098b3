"""atom_b200 -- H100 (sm_90a) implementation of the efeslab/Atom W4A4 inference hot path.

    atom_b200.ops       operator API (mirror of punica.ops)
    atom_b200.kvcache   paged INT4 KV pool (mirror of punica.utils.kvcache)
    atom_b200.llama     LinearInt4 / LlamaRMSNormInt4 / LlamaAttention / LlamaMLP / LlamaDecoderLayer
    atom_b200.qlinear   QLinearLayer surface of model/qLinearLayer.py with a real-INT4 pack()
"""
__version__ = "0.1.0"
