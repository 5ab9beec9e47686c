"""The S = 512 parity case, registered next to the cases of tests/realdims.py.

BERT-base at the longest sequence its position table allows: 2 queries + 4 contexts (1 hard negative each), lengths
~ U{128..512}, sequence 0 at full length so that position 511 is used.  The weights, batch recipe and golden format are
those of tests/realdims.py; importing this module adds the case to `realdims.CASES`, so every helper that looks a case
up by name (realdims.batch, tests/test_realdims_gpu._check_step, tests/golden/make_golden_realdims.run_case) takes it.
"""
from tests import realdims

NAME = "bert_base_s512"
CASE = ("bert", realdims.BERT_BASE, 2, 1, 512, 1.0)

realdims.CASES.setdefault(NAME, CASE)
assert realdims.CASES[NAME] == CASE, realdims.CASES[NAME]
