"""Puts the unmodified reference package (myscience/open-genie, pure Python) into oracle/_ref/ (git-ignored), so that
bench.py's CPU arm and `bench.py --impl reference` run the reference itself, also on machines without a checkout of it.

The checkout is found through OPEN_GENIE_REFERENCE, else as a sibling directory of this repository named `open-genie`
or `reference`. Nothing is installed: the `genie` package is copied, and it imports through the `lightning` stand-in
of oracle/_shim. Without a checkout (and without an earlier copy) this does nothing, and the CPU arm times the oracle
port instead, reporting kind 'oracle'.

    python oracle/vendor_reference.py            # also run by __graft_entry__.build()
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, 'oracle', '_ref')


def find_reference():
    cands = [os.environ.get('OPEN_GENIE_REFERENCE')] + [os.path.join(os.path.dirname(ROOT), n)
                                                        for n in ('open-genie', 'reference')]
    for c in cands:
        if c and os.path.isfile(os.path.join(c, 'genie', '__init__.py')):
            return c
    return None


def vendor() -> str:
    """Returns the directory that holds the copied `genie` package, or '' when no reference is available."""
    src = find_reference()
    if src is None:
        return DST if os.path.isdir(os.path.join(DST, 'genie')) else ''
    tmp = DST + '.tmp'
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(os.path.join(src, 'genie'), os.path.join(tmp, 'genie'),
                    ignore=shutil.ignore_patterns('__pycache__', '*.pyc', '.git'))
    shutil.rmtree(DST, ignore_errors=True)
    os.replace(tmp, DST)
    return DST


if __name__ == '__main__':
    print(vendor() or 'no reference checkout found', file=sys.stderr)
