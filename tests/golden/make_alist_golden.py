"""Copy the reference's WiMAX (576, 288) LDPC code description (test/codes/ldpc/wimax_576_0.5.alist) here, unchanged.
Data only.

    python tests/golden/make_alist_golden.py [REFERENCE_ROOT]
"""
import os
import shutil
import sys

ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
name = "wimax_576_0.5.alist"
shutil.copyfile(os.path.join(ref, "test", "codes", "ldpc", name),
                os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
