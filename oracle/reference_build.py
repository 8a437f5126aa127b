"""Recipe for the artefacts derived from the upstream watsor project (asmirnou/watsor) that some tests compare against.

The upstream checkout is the directory named by the environment variable WATSOR_REFERENCE, else the first of
DEFAULT_LOCATIONS that exists: a directory called `reference` beside this repository, or /root/reference.  From it
`build()` makes, under oracle/_ref/ (git-ignored):

* MODEL_DIR/b200.wb200 -- the compiled model blob of the upstream test model watsor/test/model/cpu.pb (SSD-MobileNet-v1,
  3 classes, real weights; 22 MB, too large to keep in the repository);
* REF_SITE -- an unmodified copy of the upstream `watsor` package (Python sources, no model files), whose
  `watsor.stream` runtime hosts the drop-in detector worker and whose output effects run beside the GPU effects in
  the integration tests.

Where the upstream checkout is absent nothing is built, and the tests that need these artefacts skip.
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'oracle', '_ref')
MODEL_DIR = os.path.join(OUT, 'ssd_mobilenet_v1_shapes')
MODEL_BLOB = os.path.join(MODEL_DIR, 'b200.wb200')
REF_SITE = os.path.join(OUT, 'site')


DEFAULT_LOCATIONS = (os.path.join(os.path.dirname(ROOT), 'reference'), '/root/reference')


def reference_dir():
    if os.environ.get('WATSOR_REFERENCE'):
        return os.environ['WATSOR_REFERENCE']
    for d in DEFAULT_LOCATIONS:
        if os.path.isdir(d):
            return d
    return DEFAULT_LOCATIONS[0]


def reference_pb():
    return os.path.join(reference_dir(), 'watsor', 'test', 'model', 'cpu.pb')


def has_reference():
    return os.path.isfile(os.path.join(reference_dir(), 'watsor', 'stream', 'work.py'))


def build():
    pb = reference_pb()
    if os.path.isfile(pb):
        from watsor_b200.model import compile_frozen_graph
        os.makedirs(MODEL_DIR, exist_ok=True)
        blob = compile_frozen_graph(pb, name='ssd_mobilenet_v1_shapes (watsor/test/model/cpu.pb)').to_blob()
        if not os.path.isfile(MODEL_BLOB) or open(MODEL_BLOB, 'rb').read() != blob:
            with open(MODEL_BLOB, 'wb') as f:
                f.write(blob)
    if has_reference() and not os.path.isfile(os.path.join(REF_SITE, 'watsor', 'stream', 'work.py')):
        # a plain copy of the pure-Python package: no build step, works for any user who can read the checkout
        tmp = REF_SITE + '.tmp'
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(os.path.join(reference_dir(), 'watsor'), os.path.join(tmp, 'watsor'),
                        ignore=shutil.ignore_patterns('*.pb', '__pycache__'))
        shutil.rmtree(REF_SITE, ignore_errors=True)
        os.rename(tmp, REF_SITE)
