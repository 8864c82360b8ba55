"""Model containers for the CNN operator (the ``keras.models.load_model`` +
``predict`` seam, inaSpeechSegmenter/segmenter.py:129-133,163).

The reference's three networks exist only as Keras HDF5 files fetched at run
time (remote_utils.py:4-27); their architecture is not in the source tree.
So this module (1) lowers a Keras ``model_config`` (Sequential, channels_last)
plus its weight arrays to the flat ``iss_layer_desc`` list + one float32 blob
the C ABI takes, fusing Conv2D/Dense -> BatchNormalization -> Activation
chains into GEMM epilogues, (2) reads such a model from a Keras ``.hdf5`` file
(``keras_hdf5.py``) or from an ``.npz`` with the same content, and (3) can
generate synthetic-weight stand-ins of the same family so tests and benchmarks
run without the release assets.
"""
import json
import os

import numpy as np

from . import _lib

MODEL_DIR_ENV = 'ISS_B200_MODEL_DIR'
KERAS_CACHE_DIRS = ('/root/.keras/inaSpeechSegmenter', os.path.expanduser('~/.keras/inaSpeechSegmenter'))


# --------------------------------------------------------------------------- lowering

def _same_pad(size, k, s):
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def _wget(weights, lname, var):
    for key in ('%s/%s' % (lname, var), '%s/%s:0' % (lname, var)):
        if key in weights:
            return np.asarray(weights[key], dtype=np.float32)
    for key in weights:                        # keras 2.x nests: '<layer>/<layer>/<var>:0'
        if key.endswith('/%s:0' % var) or key.endswith('/' + var):
            if key.split('/')[0] == lname:
                return np.asarray(weights[key], dtype=np.float32)
    raise KeyError('weight %s/%s not found' % (lname, var))


class LoweredModel:
    """descs: list of dicts (iss_layer_desc fields), blob: float32 array."""

    def __init__(self, descs, blob, in_h, in_w, n_classes, config, weights):
        self.descs, self.blob = descs, blob
        self.in_h, self.in_w, self.n_classes = in_h, in_w, n_classes
        self.config, self.weights = config, weights

    def c_descs(self):
        arr = (_lib.LayerDesc * len(self.descs))()
        for i, d in enumerate(self.descs):
            for k, v in d.items():
                setattr(arr[i], k, int(v))
        return arr


def lower_keras_model(config, weights, in_h, in_w, allow_no_head=False):
    """Keras Sequential config (dict / JSON) + weights -> LoweredModel.

    Supported layers: InputLayer, Conv2D, BatchNormalization, Activation /
    ReLU / Softmax, MaxPooling2D, Dropout-family (identity at inference),
    Flatten, Dense.  Anything else raises NotImplementedError naming the layer
    (no silent approximation)."""
    if isinstance(config, (str, bytes)):
        config = json.loads(config)
    cfg = config.get('config', config)
    layers = cfg['layers'] if isinstance(cfg, dict) else cfg
    blob, descs = [], []
    pos = [0]

    def push(a):
        a = np.ascontiguousarray(a, dtype=np.float32).ravel()
        off = pos[0]
        blob.append(a)
        pad = (-len(a)) % 4                   # keep every tensor 16-byte aligned for float4 loads
        if pad:
            blob.append(np.zeros(pad, np.float32))
        pos[0] += len(a) + pad
        return off

    def new_desc(kind):
        return dict(kind=kind, kh=1, kw=1, sh=1, sw=1, pad_top=0, pad_left=0, pad_bottom=0, pad_right=0,
                    cin=0, cout=0, flags=0, w_off=-1, bias_off=-1, pre_scale_off=-1, pre_shift_off=-1,
                    post_scale_off=-1, post_shift_off=-1)

    h, w, c = in_h, in_w, 1
    flat = False
    cur = None                 # the GEMM-like layer whose epilogue can still absorb ops
    softmax_layers = []        # iss_cnn_forward honours softmax on the head only

    def apply_act(name):
        nonlocal cur
        if name in (None, 'linear'):
            return
        if cur is None:
            raise NotImplementedError('activation %r without a preceding Conv2D/Dense' % name)
        # the kernels' epilogue order is fixed: bias -> affine(pre) -> ReLU -> sigmoid -> affine(post); anything a
        # model asks for in another order is refused rather than silently reordered
        if name == 'relu':
            if cur['flags'] & (_lib.F_RELU | _lib.F_SIGMOID | _lib.F_AFFINE_POST | _lib.F_SOFTMAX):
                raise NotImplementedError('activation chain too long to fuse')
            cur['flags'] |= _lib.F_RELU
        elif name == 'softmax':
            if cur['flags'] & (_lib.F_RELU | _lib.F_SIGMOID | _lib.F_AFFINE_POST | _lib.F_SOFTMAX):
                raise NotImplementedError('softmax after another activation')
            cur['flags'] |= _lib.F_SOFTMAX
            softmax_layers.append(cur)
            cur = None
        elif name == 'sigmoid':
            if cur['flags'] & (_lib.F_SIGMOID | _lib.F_AFFINE_POST | _lib.F_SOFTMAX):
                raise NotImplementedError('sigmoid after an activation the epilogue evaluates later')
            cur['flags'] |= _lib.F_SIGMOID
        else:
            raise NotImplementedError('activation %r' % name)

    for layer in layers:
        cls, lc = layer['class_name'], layer['config']
        name = lc.get('name')
        if cls in ('InputLayer', 'Dropout', 'SpatialDropout2D', 'GaussianNoise', 'GaussianDropout'):
            continue
        if cls == 'Conv2D':
            if flat:
                raise NotImplementedError('Conv2D after Flatten')
            if tuple(lc.get('dilation_rate', (1, 1))) != (1, 1) or lc.get('groups', 1) != 1:
                raise NotImplementedError('dilated / grouped Conv2D')
            if lc.get('data_format', 'channels_last') != 'channels_last':
                raise NotImplementedError('channels_first')
            k = _wget(weights, name, 'kernel')
            kh, kw, cin, cout = k.shape
            assert cin == c, (name, cin, c)
            d = new_desc(_lib.LAYER_CONV2D)
            sh, sw = lc.get('strides', (1, 1))
            d.update(kh=kh, kw=kw, sh=sh, sw=sw, cin=cin, cout=cout, w_off=push(k))
            if lc.get('padding', 'valid') == 'same':
                d['pad_top'], d['pad_bottom'] = _same_pad(h, kh, sh)
                d['pad_left'], d['pad_right'] = _same_pad(w, kw, sw)
            if lc.get('use_bias', True):
                d['flags'] |= _lib.F_BIAS
                d['bias_off'] = push(_wget(weights, name, 'bias'))
            h = (h + d['pad_top'] + d['pad_bottom'] - kh) // sh + 1
            w = (w + d['pad_left'] + d['pad_right'] - kw) // sw + 1
            c = cout
            descs.append(d)
            cur = d
            apply_act(lc.get('activation'))
        elif cls == 'Dense':
            k = _wget(weights, name, 'kernel')
            cin, cout = k.shape
            assert cin == h * w * c, (name, cin, h, w, c)
            d = new_desc(_lib.LAYER_DENSE)
            d.update(cin=cin, cout=cout, w_off=push(k))
            if lc.get('use_bias', True):
                d['flags'] |= _lib.F_BIAS
                d['bias_off'] = push(_wget(weights, name, 'bias'))
            h, w, c, flat = 1, 1, cout, True
            descs.append(d)
            cur = d
            apply_act(lc.get('activation'))
        elif cls == 'BatchNormalization':
            if cur is None:
                raise NotImplementedError('BatchNormalization without a preceding Conv2D/Dense')
            axis = lc.get('axis', -1)
            axis = axis[0] if isinstance(axis, (list, tuple)) else axis
            if axis not in (-1, 3, 1 if flat else 3):
                raise NotImplementedError('BatchNormalization axis %r' % (axis,))
            eps = lc.get('epsilon', 1e-3)
            mean = _wget(weights, name, 'moving_mean').astype(np.float32)
            var = _wget(weights, name, 'moving_variance').astype(np.float32)
            inv = (1.0 / np.sqrt(var + np.float32(eps))).astype(np.float32)
            scale = inv * _wget(weights, name, 'gamma') if lc.get('scale', True) else inv
            shift = (_wget(weights, name, 'beta') if lc.get('center', True) else np.float32(0)) - mean * scale
            scale, shift = scale.astype(np.float32), np.broadcast_to(shift, scale.shape).astype(np.float32)
            if not cur['flags'] & (_lib.F_RELU | _lib.F_SIGMOID | _lib.F_AFFINE_PRE):
                cur['flags'] |= _lib.F_AFFINE_PRE
                cur['pre_scale_off'], cur['pre_shift_off'] = push(scale), push(shift)
            elif not cur['flags'] & _lib.F_AFFINE_POST:
                cur['flags'] |= _lib.F_AFFINE_POST
                cur['post_scale_off'], cur['post_shift_off'] = push(scale), push(shift)
            else:
                raise NotImplementedError('more than two BatchNormalization layers after one Conv2D/Dense')
        elif cls == 'Activation':
            apply_act(lc['activation'])
        elif cls == 'ReLU':
            apply_act('relu')
        elif cls == 'Softmax':
            apply_act('softmax')
        elif cls == 'MaxPooling2D':
            ph, pw = lc.get('pool_size', (2, 2))
            st = lc.get('strides') or (ph, pw)
            d = new_desc(_lib.LAYER_MAXPOOL)
            d.update(kh=ph, kw=pw, sh=st[0], sw=st[1], cin=c, cout=c)
            if lc.get('padding', 'valid') == 'same':
                d['pad_top'], d['pad_bottom'] = _same_pad(h, ph, st[0])
                d['pad_left'], d['pad_right'] = _same_pad(w, pw, st[1])
            h = (h + d['pad_top'] + d['pad_bottom'] - ph) // st[0] + 1
            w = (w + d['pad_left'] + d['pad_right'] - pw) // st[1] + 1
            descs.append(d)
            cur = None
        elif cls == 'Flatten':
            flat = True                     # NHWC memory order == Keras channels_last flatten order
            cur = None
        else:
            raise NotImplementedError('Keras layer %s is not supported by the GPU CNN operator' % cls)
    if any(d is not descs[-1] for d in softmax_layers):
        raise NotImplementedError('softmax on a layer that is not the head')
    if not (h == 1 and w == 1) and not (allow_no_head and flat):
        raise NotImplementedError('model must end in a Dense head')
    return LoweredModel(descs, np.concatenate(blob) if blob else np.zeros(0, np.float32), in_h, in_w, c,
                        config, weights)


# --------------------------------------------------------------------------- synthetic stand-ins

def synthetic_keras_cnn(nmel, n_classes, seed=0, width=1.0):
    """A Keras-style Sequential of the family the reference papers describe
    (4 Conv2D + BN + ReLU blocks with two 2x2 max-poolings, then Dense + BN +
    ReLU blocks and a softmax head; ~1.4 M parameters like the ~5 MB release
    files).  Weights are seeded He-normal, BatchNorm statistics are random but
    well conditioned.  This is a STAND-IN: the real architecture ships only
    inside keras_*_cnn.hdf5."""
    rng = np.random.default_rng(seed)
    c1, c2, d1 = int(64 * width), int(128 * width), int(512 * width)
    layers, weights = [], {}
    idx = [0]

    def uid(prefix):
        idx[0] += 1
        return '%s_%d' % (prefix, idx[0])

    def bn(ch):
        n = uid('batch_normalization')
        weights[n + '/gamma'] = rng.uniform(0.8, 1.2, ch).astype(np.float32)
        weights[n + '/beta'] = rng.normal(0, 0.1, ch).astype(np.float32)
        weights[n + '/moving_mean'] = rng.normal(0, 0.2, ch).astype(np.float32)
        weights[n + '/moving_variance'] = rng.uniform(0.5, 1.5, ch).astype(np.float32)
        layers.append({'class_name': 'BatchNormalization', 'config': {'name': n, 'axis': [3], 'epsilon': 1e-3,
                                                                      'center': True, 'scale': True}})

    def act(a):
        layers.append({'class_name': 'Activation', 'config': {'name': uid('activation'), 'activation': a}})

    def conv(cin, cout, kh, kw):
        n = uid('conv2d')
        weights[n + '/kernel'] = (rng.standard_normal((kh, kw, cin, cout)) * np.sqrt(2.0 / (kh * kw * cin))).astype(np.float32)
        weights[n + '/bias'] = rng.normal(0, 0.05, cout).astype(np.float32)
        layers.append({'class_name': 'Conv2D', 'config': {'name': n, 'filters': cout, 'kernel_size': [kh, kw],
                                                          'strides': [1, 1], 'padding': 'valid', 'use_bias': True,
                                                          'activation': 'linear', 'data_format': 'channels_last'}})
        bn(cout)
        act('relu')

    def pool():
        layers.append({'class_name': 'MaxPooling2D', 'config': {'name': uid('max_pooling2d'), 'pool_size': [2, 2],
                                                                'strides': [2, 2], 'padding': 'valid'}})

    def dense(cin, cout, last=False):
        n = uid('dense')
        weights[n + '/kernel'] = (rng.standard_normal((cin, cout)) * np.sqrt((1.0 if last else 2.0) / cin)).astype(np.float32)
        weights[n + '/bias'] = rng.normal(0, 0.05, cout).astype(np.float32)
        layers.append({'class_name': 'Dense', 'config': {'name': n, 'units': cout, 'use_bias': True,
                                                         'activation': 'softmax' if last else 'linear'}})
        if not last:
            bn(cout)
            act('relu')
            layers.append({'class_name': 'Dropout', 'config': {'name': uid('dropout'), 'rate': 0.2}})

    layers.append({'class_name': 'InputLayer', 'config': {'name': 'input_1', 'batch_input_shape': [None, 68, nmel, 1]}})
    h, w = 68, nmel
    conv(1, c1, 4, 5);   h, w = h - 3, w - 4
    conv(c1, c1, 5, 4);  h, w = h - 4, w - 3
    pool();              h, w = h // 2, w // 2
    conv(c1, c2, 3, 3);  h, w = h - 2, w - 2
    conv(c2, c2, 3, 3);  h, w = h - 2, w - 2
    pool();              h, w = h // 2, w // 2
    layers.append({'class_name': 'Flatten', 'config': {'name': 'flatten_1'}})
    dense(h * w * c2, d1)
    dense(d1, d1)
    dense(d1, n_classes, last=True)
    config = {'class_name': 'Sequential', 'config': {'name': 'sequential_1', 'layers': layers}}
    return config, weights


def save_npz(path, config, weights):
    np.savez(path, model_config=np.array(json.dumps(config)), **{'w:' + k: v for k, v in weights.items()})


def load_npz(path):
    z = np.load(path, allow_pickle=False)
    config = json.loads(str(z['model_config']))
    weights = {k[2:]: z[k] for k in z.files if k.startswith('w:')}
    return config, weights


def find_model_file(fname):
    """Model lookup order: $ISS_B200_MODEL_DIR, then the reference's own
    convention /root/.keras/inaSpeechSegmenter/<f> and ~/.keras/... (remote_utils.py:18-27).
    No download is attempted (no network on the target boxes)."""
    dirs = [os.environ[MODEL_DIR_ENV]] if os.environ.get(MODEL_DIR_ENV) else []
    for d in dirs + list(KERAS_CACHE_DIRS):
        for cand in (fname, os.path.splitext(fname)[0] + '.npz'):
            p = os.path.join(d, cand)
            if os.access(p, os.R_OK):
                return p
    return None


def load_model_file(path):
    if path.endswith('.npz'):
        return load_npz(path)
    from . import keras_hdf5
    return keras_hdf5.load_keras_hdf5(path)
