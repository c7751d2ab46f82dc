"""Runs the reference built into oracle/_ref (see make_ref.py) on CPU: its own model.yolo2.Darknet, model.Inference, F.softmax and
detect.postprocess -- the chain of detect.py:141-153 for a batch -- for the CPU arm of bench.py.  Must be imported in a process that
has NOT imported this repository's own `model` / `utils` packages (the reference uses the same top-level names)."""
import configparser
import marshal
import os
import sys
import types
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(HERE, '_ref')


def available():
    return os.path.isfile(os.path.join(REFDIR, 'model', 'yolo2.pyc')) and os.path.isfile(os.path.join(REFDIR, 'detect.pyc'))


def load():
    """Import the reference's modules from oracle/_ref.  detect.py itself cannot be imported (humanize / pybenchmark / cv2 GUI
    imports at detect.py:28-32), so its three pure functions on the path are taken from its compiled module's constants."""
    import torch
    warnings.filterwarnings('ignore')
    if 'model' in sys.modules or 'utils' in sys.modules:
        raise RuntimeError('ref_runner: `model` / `utils` already imported from elsewhere')
    sys.path.insert(0, REFDIR)
    import model  # noqa: F401
    import model.yolo2  # noqa: F401
    import utils  # noqa: F401
    import utils.postprocess  # noqa: F401
    with open(os.path.join(REFDIR, 'detect.pyc'), 'rb') as f:
        module_code = marshal.loads(f.read()[16:])
    pyb = types.SimpleNamespace(profile=lambda name: (lambda fn: fn))       # detect.py's timing decorator, a no-op here
    ns = dict(torch=torch, utils=sys.modules['utils'], pybenchmark=pyb)
    fns = {c.co_name: types.FunctionType(c, ns, c.co_name) for c in module_code.co_consts
           if isinstance(c, types.CodeType) and c.co_name in ('get_logits', 'filter_visible', 'postprocess')}
    ns.update(fns)
    return sys.modules['model'], types.SimpleNamespace(**fns)


def build_chain(state_dict, anchors):
    """Returns chain(x[B,3,H,W]) -> (feature, [per-image detect.postprocess result])."""
    import torch
    model, detect = load()
    config = configparser.ConfigParser()
    config.read_dict({'batch_norm': {'enable': '1'}, 'detect': {'threshold': '0.3', 'threshold_cls': '0.005', 'fix': '1', 'overlap': '0.45'}})
    dnn = model.yolo2.Darknet(model.ConfigChannels(config), anchors, 20)
    dnn.load_state_dict(state_dict, strict=False)
    dnn.eval()
    inference = model.Inference(config, dnn, anchors)
    inference.eval()

    def chain(x):
        with torch.no_grad():
            pred = model._inference(inference, x)
            prob = torch.nn.functional.softmax(detect.get_logits(pred), -1)
            out = []
            for bi in range(x.size(0)):
                iou, yx_min, yx_max, p = (t[bi].reshape(-1, *t.shape[3:]) if t.dim() > 3 else t[bi].reshape(-1)
                                          for t in (pred['iou'], pred['yx_min'], pred['yx_max'], prob))
                out.append(detect.postprocess(config, iou, yx_min, yx_max, p))
        return pred['feature'], out

    return chain
