"""Import shim: `from ringattention import ringattention, blockwise_feedforward, ringattention_jax,
ringattention_inference` (lwm/llama.py:30) resolves to the H100 ops."""
from lwm_b200.blockwise_ffn import blockwise_feedforward  # noqa: F401
from lwm_b200.ringattention import ringattention, ringattention_inference, set_axis_group  # noqa: F401

ringattention_jax = ringattention      # the reference picks the pure-JAX variant off-TPU (llama.py:538); same op here
