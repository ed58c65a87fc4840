"""Run the reference's own model code on deephar_b200 without editing it.

    import deephar_b200.dropin
    deephar_b200.dropin.install()                # before the first `import deephar` / `import keras`
    sys.path.insert(0, '/path/to/deephar')       # the reference checkout
    from deephar.models import reception, spnet
    model = reception.build(input_shape, 16, dim=2, num_blocks=8, num_context_per_joint=2, ksize=(5, 5))
    model.load_weights('weights_PE_MPII_cvpr18_19-09-2017.h5')
    pred = model.predict(frames)                 # sm_90a kernels

`install()` registers a `keras` package (and a `tensorflow` stand-in) in `sys.modules` whose layer classes are
keras_compat's and whose backend is keras_trace's: the reference's builders (deephar/models/reception.py, spnet.py,
common.py on its own layers.py / activations.py / config.py) then RECORD deephar_b200's layer graph instead of building a
TensorFlow graph, and the `Model(...)` they return is the compiled H100 model with the `keras.Model` protocol the
evaluators use; `spnet.split_model` and `action.build_merge_model(model_pe, ...)` (get_layer / TimeDistributed re-wiring
of the pose network, action.py:112-400) work on those models the same way.  The four parameter-free head-model builders of deephar/models/blocks.py:217-343 (soft-argmax 2-D / 1-D,
joint probability, context aggregation -- frozen Dense / SeparableConv2D / tf.divide sub-models in the reference) are
provided here as recordable objects under the module name `deephar.models.blocks`.

Everything the reference merely imports but the forward path never calls -- optimizers, callbacks, regularizers, losses,
data utilities, the unused layer classes -- exists as an inert stand-in, or as a stub that raises NotImplementedError
naming itself when it is called: training stays with the reference.  tests/test_keras_compat.py holds the evidence: the
models recorded this way for every BASELINE configuration are deephar_b200's own, expression for expression.
"""
import sys
import types

from . import keras_compat, keras_trace

_BACKEND = ('int_shape', 'ndim', 'epsilon', 'image_data_format', 'set_image_data_format', 'expand_dims', 'squeeze', 'tile',
            'sum', 'mean', 'max', 'exp', 'clip', 'stop_gradient', 'reshape')
_LAYERS = ('Activation', 'Add', 'AveragePooling2D', 'BatchNormalization', 'Concatenate', 'Conv2D', 'GlobalMaxPooling1D',
           'GlobalMaxPooling2D', 'Input', 'Lambda', 'MaxPooling2D', 'Multiply', 'SeparableConv2D', 'TimeDistributed',
           'UpSampling2D', 'ZeroPadding2D', 'add', 'concatenate', 'multiply')
_HEADS = ('build_context_aggregation', 'build_joints_probability', 'build_softargmax_1d', 'build_softargmax_2d')


def _module(name, doc, **members):
    m = types.ModuleType(name, doc)
    m.__dict__.update(members)
    return m


def _stubbed(mod, what):
    """Any other attribute of `mod` is a callable that fails, when called, with the name of what is missing."""
    def missing(attr):
        if attr.startswith('__'):
            raise AttributeError(attr)

        def stub(*args, **kwargs):
            raise NotImplementedError('%s.%s is not part of the recording front end (deephar_b200.keras_compat): only '
                                      'the forward path of the reference models is' % (what, attr))
        stub.__name__ = attr
        return stub
    mod.__getattr__ = missing
    return mod


class _Inert(object):
    """Optimizers, callbacks, ...: constructed by training code the forward path never runs."""

    def __init__(self, *args, **kwargs):
        pass


def get_file(fname, origin=None, untar=False, md5_hash=None, file_hash=None, cache_subdir='datasets',
             hash_algorithm='auto', extract=False, archive_format='auto', cache_dir=None):
    """keras.utils.data_utils.get_file for the case the reference's scripts rely on after their first run: the file is
    already in the Keras cache (`~/.keras/<cache_subdir>/<fname>`, or `fname` itself when it is an absolute path --
    exp/mpii/eval_mpii_singleperson.py:51-53, datasets/annothelper.py:12-14) and its path is returned.  Nothing is ever
    downloaded: a missing file is an error that says where to put it.  A hash that differs from the published one is
    reported, and the local file is used (Keras would download it again)."""
    import hashlib
    import os
    import warnings
    if untar or extract:
        raise NotImplementedError('keras.utils.data_utils.get_file: archives are not unpacked here')
    base = os.path.expanduser(cache_dir or os.environ.get('KERAS_HOME') or os.path.join('~', '.keras'))
    path = os.path.join(base, cache_subdir, fname)
    if not os.path.exists(path):
        raise IOError('keras.utils.data_utils.get_file: %s is not there and nothing is downloaded; fetch %s and place '
                      'it at that path' % (path, origin))
    want = file_hash or md5_hash
    if want:
        algo = 'md5' if (hash_algorithm == 'md5' or (hash_algorithm == 'auto' and len(want) == 32)) else 'sha256'
        h = hashlib.new(algo)
        with open(path, 'rb') as f:
            for chunk in iter(lambda: f.read(1 << 20), b''):
                h.update(chunk)
        if h.hexdigest() != want:
            warnings.warn('%s: %s %s differs from the published %s; using the local file' % (path, algo, h.hexdigest(), want))
    return path


def install(override_blocks=True):
    """Register the recording `keras` / `tensorflow` (idempotent).  Refuses to replace a real Keras that is already
    imported.  Returns the `keras` module."""
    have = sys.modules.get('keras')
    if have is not None:
        if getattr(have, '__deephar_b200__', False):
            return have
        raise RuntimeError('a real `keras` is already imported; call deephar_b200.dropin.install() first')

    keras = _module('keras', 'keras -> deephar_b200.keras_compat (recording front end)', __version__='2.1.4',
                    __deephar_b200__=True, __path__=[])
    backend = _stubbed(_module('keras.backend', 'keras.backend -> deephar_b200.keras_trace',
                               **{k: getattr(keras_trace, k) for k in _BACKEND}), 'keras.backend')
    backend.clear_session = keras_compat.clear_session
    layers = _stubbed(_module('keras.layers', 'keras.layers -> deephar_b200.keras_compat',
                              **{k: getattr(keras_compat, k) for k in _LAYERS}), 'keras.layers')
    models = _stubbed(_module('keras.models', 'keras.models -> deephar_b200.keras_compat', Model=keras_compat.Model),
                      'keras.models')
    inert = lambda *names: {n: type(n, (_Inert,), {}) for n in names}       # noqa: E731
    optimizers = _module('keras.optimizers', 'inert', **inert('SGD', 'RMSprop', 'Adam'))
    callbacks = _module('keras.callbacks', 'inert',
                        **inert('Callback', 'LearningRateScheduler', 'ProgbarLogger', 'TensorBoard', 'ModelCheckpoint'))
    nothing = lambda *a, **k: None                                          # noqa: E731
    regularizers = _module('keras.regularizers', 'inert', l1=nothing, l2=nothing)
    constraints = _module('keras.constraints', 'inert', unit_norm=nothing)
    losses = _stubbed(_module('keras.losses', 'training only'), 'keras.losses')
    data_utils = _module('keras.utils.data_utils', 'cache look-up only, no network', get_file=get_file)
    utils = _module('keras.utils', 'inert', data_utils=data_utils, __path__=[], **inert('Sequence', 'OrderedEnqueuer'))
    tensorflow = _stubbed(_module('tensorflow', 'tensorflow stand-in: nothing of it is on the recorded forward path',
                                  __version__='1.6.0'), 'tensorflow')

    keras.backend, keras.layers, keras.models, keras.optimizers, keras.callbacks = backend, layers, models, optimizers, callbacks
    keras.regularizers, keras.constraints, keras.losses, keras.utils = regularizers, constraints, losses, utils
    registry = {'keras': keras, 'keras.backend': backend, 'keras.layers': layers, 'keras.models': models,
                'keras.optimizers': optimizers, 'keras.callbacks': callbacks, 'keras.regularizers': regularizers,
                'keras.constraints': constraints, 'keras.losses': losses, 'keras.utils': utils,
                'keras.utils.data_utils': data_utils}
    if 'tensorflow' not in sys.modules:
        registry['tensorflow'] = tensorflow
    if override_blocks:
        registry['deephar.models.blocks'] = _module(
            'deephar.models.blocks', 'deephar/models/blocks.py:217-343 as recordable head models (deephar_b200.keras_compat)',
            **{k: getattr(keras_compat, k) for k in _HEADS})
    sys.modules.update(registry)
    return keras


def uninstall():
    """Remove what install() registered (and the reference modules that were imported on top of it)."""
    if not getattr(sys.modules.get('keras'), '__deephar_b200__', False):
        return
    for name in list(sys.modules):
        root = name.split('.')[0]
        if root in ('keras', 'deephar') or (root == 'tensorflow' and sys.modules[name].__doc__
                                            and 'stand-in' in sys.modules[name].__doc__):
            del sys.modules[name]
