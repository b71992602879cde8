"""CPU oracle — TEST INFRASTRUCTURE ONLY.

Restatements of the reference algorithms used solely as checkers by tests/, by
__graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference legs. Nothing under
lwm_b200/ may import this package: the product path is the CUDA library or a loud failure.

PARITY STATUS
  * VQGAN: PINNED (structure) — tests/golden/vqgan_reference_small.npz is produced by executing the UNMODIFIED
    reference module lwm/vqgan.py over a numpy-backed shim of its jax/flax/tux imports
    (oracle/flax_shim, tools/make_golden_vqgan_from_reference.py); oracle/vqgan_ref.py reproduces it (indices
    bit-exact, floats to 1e-6). The semantics of the flax primitives themselves (nn.Conv SAME/HWIO, nn.GroupNorm
    defaults, nearest resize) are this repo's reading of flax 0.8.4 — not executable offline.
  * RoPE (oracle/rope.py) and vision token framing (oracle/vision_tokens.py): PINNED — fixtures produced by executing
    the reference's own functions / class (source text extracted at generation time from lwm/llama.py and lwm/data.py,
    tools/make_golden_next_rows_from_reference.py); reproduced bit for bit.
  * Ring attention: UNPINNED — see below.
PARITY UNPINNED (ring attention): the reference ships no tests / golden vectors, the ring-attention arithmetic
lives in the un-vendored, un-pinned `ringattention` pip package (gpu_requirements.txt:8), and
jax/flax cannot be imported in the build container (no network, wheelhouse excludes jax), so the
oracle could not be checked against outputs of the reference itself. It is pinned instead against
(a) an independent dense fp64 formulation, (b) torch's own CPU operators
(scaled_dot_product_attention / conv2d / group_norm) and (c) mathematical invariants — see
tests/test_oracle_*.py and DESIGN.md.
"""
