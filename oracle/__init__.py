"""CPU oracle: plain PyTorch fp32 restatements of the reference algorithms on the SEED-X hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under seed-x_b200/ (the product) imports this package; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use it, as the checker or the timed
CPU baseline.  Each function cites the reference file:line it restates.  Pinning status per module is stated in each
module header (golden vectors generated from the reference itself live in tests/golden/).
"""
