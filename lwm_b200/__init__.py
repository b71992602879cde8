"""lwm_b200 — H100 (sm_90a) native hot paths of LargeWorldModel/LWM.

Two paths only (SURVEY.md §8): the blockwise RingAttention operator called in
`FlaxLLaMAAttention.__call__` (lwm/llama.py:539-569) and the VQGAN tokenizer (lwm/vqgan.py).
The compute lives in `lib/liblwm_b200.so` (hand-written CUDA, C ABI in include/lwm_b200.h);
this package is the thin host-side mirror of the reference's Python operator signatures.
There is no CPU fallback: importing works anywhere, calling an op needs an sm_90 GPU.
"""
__version__ = "0.1.0"
