#!/usr/bin/env python
"""Build the reference arm of bench.py (`--impl reference`, `cpu_baseline.kind = "reference"`) into oracle/_ref/.

The reference (ruiminshen/yolo2-pytorch) is a script tree without setup.py / pyproject.toml, so `pip install` cannot install
it.  This compiles the modules on its hot path -- model/, utils/ and detect.py -- to Python bytecode and writes only the
compiled files to `oracle/_ref/` (git-ignored), as sourceless modules that `import model.yolo2` etc. load directly.  One line is
changed before compiling: `utils/__init__.py:109` names a parameter `async`, a reserved word since Python 3.7, so nothing
compiles without the rename to `non_blocking`.  `__graft_entry__.build()` runs this when the reference checkout is readable
(`YB_REFERENCE_DIR`, default /root/reference); otherwise whatever oracle/_ref/ already holds is kept.

    python oracle/make_ref.py
"""
import importlib.util
import marshal
import os
import shutil
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('YB_REFERENCE_DIR', '/root/reference')
DST = os.path.join(HERE, '_ref')
PACKAGES = ('model', 'utils')
MODULES = ('detect.py',)


def _sources():
    for pkg in PACKAGES:
        for d, _, files in os.walk(os.path.join(REF, pkg)):
            for f in sorted(files):
                if f.endswith('.py'):
                    yield os.path.relpath(os.path.join(d, f), REF)
    for m in MODULES:
        yield m


def _pyc(code):
    # PEP 552 header: magic, flags = 0 (timestamp form), mtime, source size -- unused for a sourceless module
    return importlib.util.MAGIC_NUMBER + (0).to_bytes(4, 'little') + (0).to_bytes(4, 'little') + (0).to_bytes(4, 'little') + marshal.dumps(code)


def main():
    if not os.path.isfile(os.path.join(REF, 'model', 'yolo2.py')):
        return 0
    shutil.rmtree(DST, ignore_errors=True)
    for rel in _sources():
        text = open(os.path.join(REF, rel)).read()
        if rel == os.path.join('utils', '__init__.py'):
            patched = text.replace('async=False', 'non_blocking=False').replace('device_id, async)', 'device_id, non_blocking)')
            if patched == text and 'async' in text:
                raise SystemExit('make_ref: the async rename did not apply')
            text = patched
        with warnings.catch_warnings():                     # the reference's own invalid escape sequences
            warnings.simplefilter('ignore', SyntaxWarning)
            code = compile(text, os.path.join('reference', rel), 'exec', dont_inherit=True)
        out = os.path.join(DST, rel[:-3] + '.pyc')
        os.makedirs(os.path.dirname(out), exist_ok=True)
        with open(out, 'wb') as f:
            f.write(_pyc(code))
    return 0


if __name__ == '__main__':
    sys.exit(main())
