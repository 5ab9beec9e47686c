#!/usr/bin/env python3
"""Golden vectors of the S = 512 case (tests/realdims_long.py), produced by the UNMODIFIED reference with the same
machinery as make_golden_realdims.py:

  python tests/golden/make_golden_long.py          # writes tests/golden/realdims_bert_base_s512.npz  (~30 s)
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden_realdims import run_case  # noqa: E402
from tests import realdims_long  # noqa: E402

if __name__ == "__main__":
    run_case(realdims_long.NAME)
