#!/usr/bin/env python
"""Recipe that copies the UNMODIFIED LongCTR input path of the reference (reczoo/FuxiCTR),
model_zoo/LongCTR/longctr_dataloader.py, to oracle/_ref/extras/model_zoo/LongCTR/, where
tools/longctr_input_times.py times the reference's collator against the HBM store.  `__graft_entry__.build()`
calls install() after oracle/install_ref.py; by hand:

    python oracle/install_longctr_ref.py

The reference checkout is read from $FUXICTR_REFERENCE (default /root/reference).  When it is absent, a copy made
earlier is kept (a copy of the tree made after the build carries it along), and without either the timing tool
skips its reference arms.  oracle/_ref is git-ignored: nothing under it enters history.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("FUXICTR_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "model_zoo", "LongCTR", "longctr_dataloader.py")
DST = os.path.join(HERE, "_ref", "extras", "model_zoo", "LongCTR", "longctr_dataloader.py")


def install():
    """Copy the reference's longctr_dataloader.py unless it is already there.  Returns True when oracle/_ref holds
    it afterwards."""
    if os.path.exists(DST):
        return True
    if not os.path.exists(SRC):
        return False
    os.makedirs(os.path.dirname(DST), exist_ok=True)
    shutil.copyfile(SRC, DST)
    return True


if __name__ == "__main__":
    if not install():
        raise SystemExit("no reference checkout at %s (set FUXICTR_REFERENCE)" % REF)
    print("copied", SRC, "to", DST)
