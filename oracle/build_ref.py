"""Recipe that installs the unmodified reference (zgcr/SimpleAICV_pytorch_training_examples) into oracle/_ref/ for the
tests that compare with it (baseline/ref_import.py).  Its two import roots, ``SimpleAICV`` and ``tools``, are copied as
they are: the reference ships no setup.py, and nothing in it is edited.  oracle/_ref/ is git-ignored.

The reference checkout is taken from $SAICV_REFERENCE_DIR, else from /root/reference.  Without one, nothing is installed
and the live comparisons skip; tests/golden/ holds what the reference computed for the GPU parity test.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, '_ref')


def reference_dir():
    d = os.environ.get('SAICV_REFERENCE_DIR', '/root/reference')
    return d if os.path.isdir(os.path.join(d, 'SimpleAICV')) and os.path.isdir(os.path.join(d, 'tools')) else None


def install():
    """Copies the reference into oracle/_ref/ (replacing an older copy); returns the destination or None."""
    src = reference_dir()
    if src is None:
        return DEST if os.path.isdir(os.path.join(DEST, 'SimpleAICV')) else None
    tmp = DEST + '.tmp'
    shutil.rmtree(tmp, ignore_errors=True)
    for name in ('SimpleAICV', 'tools'):
        shutil.copytree(os.path.join(src, name), os.path.join(tmp, name),
                        ignore=shutil.ignore_patterns('__pycache__', '*.pyc', '*.pth', '*.pt'))
    shutil.rmtree(DEST, ignore_errors=True)
    os.replace(tmp, DEST)
    return DEST


if __name__ == '__main__':
    print(install())
