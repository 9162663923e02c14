"""unicore_b200: the Hopper (sm_90a) core under the Uni-Core compatible ``unicore`` API.

``ops``      hand-written CUDA kernels + autograd wrappers (``csrc/`` -> ``unicore_b200._C``)
``parallel`` symmetric-memory data parallel engine (peer-memory all-reduce fused with Adam)
``models``   flagship models built on the fused ops (BERT, Uni-Mol style SE(3) transformer)
``utils``    device timing, clock sampling, build helpers
"""
__version__ = "0.1.0"
