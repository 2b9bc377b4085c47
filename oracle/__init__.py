"""oracle/ -- TEST INFRASTRUCTURE ONLY.

CPU restatement (stock torch.nn + numpy) of the reference's Generator/Discriminator hot path.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package, and only as the checker or the timed CPU baseline -- never from the product path
(pytorch-gan_b200/), which fails loudly when libb200gan.so is missing.

Pinning: the reference holds no tests or golden vectors (SURVEY.md section 8c), so this oracle is
pinned against outputs of the reference itself: oracle/make_golden.py imports/executes the
reference's own Python from a checkout of the reference (no GPU needed), asserts that the restatement
reproduces it bit-for-bit on CPU, and commits small fixtures under tests/golden/.
"""
