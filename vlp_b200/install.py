"""Drop-in installation under the reference's import path.

The reference drivers import their model classes with
    from pytorch_pretrained_bert.modeling import BertForPreTrainingLossMask      (vlp/run_img2txt_dist.py:24)
    from pytorch_pretrained_bert.modeling import BertForSeq2SeqDecoder           (vlp/decode_img2txt.py:20)
`install()` makes those names resolve to the H100-native classes of vlp_b200.vlp_modules, either by rebinding them in
an already-imported reference `modeling` module or — when the reference package cannot be imported on this stack
(boto3 / torch._six / apex, SURVEY.md §8c) — by registering vlp_b200.vlp_modules itself as `pytorch_pretrained_bert.modeling`.
"""
import sys
import types

from . import vlp_modules as vm

_NAMES = ["BertConfig", "BertLayerNorm", "BertEmbeddings", "BertSelfAttention", "BertSelfOutput", "BertAttention", "BertIntermediate",
          "BertOutput", "BertLayer", "BertEncoder", "BertPooler", "BertPredictionHeadTransform", "BertLMPredictionHead",
          "BertPreTrainingHeads", "PreTrainedBertModel", "BertModel", "BertModelIncr", "BertForPreTrainingLossMask", "BertForSeq2SeqDecoder"]


def install_optimizer():
    """Opt-in: serve `from pytorch_pretrained_bert.optimization import BertAdam, warmup_linear` (run_img2txt_dist.py:25) from
    vlp_b200.optimization (fused multi-tensor step, SURVEY.md §8f-1).  The reference module cannot be imported on a modern stack
    at all (`torch._six`, optimization.py:27), so this registers rather than rebinds."""
    from . import optimization as vo
    mod = sys.modules.get("pytorch_pretrained_bert.optimization")
    if mod is not None and mod is not vo:
        for n in ("BertAdam", "SCHEDULES", "warmup_cosine", "warmup_constant", "warmup_linear"):
            setattr(mod, n, getattr(vo, n))
        return mod
    pkg = sys.modules.get("pytorch_pretrained_bert")
    if pkg is None:
        pkg = types.ModuleType("pytorch_pretrained_bert")
        pkg.__path__ = []
        sys.modules["pytorch_pretrained_bert"] = pkg
    sys.modules["pytorch_pretrained_bert.optimization"] = vo
    pkg.optimization = vo
    return vo


def install(shadow=True, optimizer=False):
    """Rebind the hot-path classes.  Returns the module object now serving `pytorch_pretrained_bert.modeling`."""
    if optimizer:
        install_optimizer()
    mod = sys.modules.get("pytorch_pretrained_bert.modeling")
    if mod is not None and mod is not vm:
        for n in _NAMES:
            setattr(mod, n, getattr(vm, n))
        return mod
    if shadow:
        pkg = sys.modules.get("pytorch_pretrained_bert")
        if pkg is None:
            pkg = types.ModuleType("pytorch_pretrained_bert")
            pkg.__path__ = []
            sys.modules["pytorch_pretrained_bert"] = pkg
        sys.modules["pytorch_pretrained_bert.modeling"] = vm
        pkg.modeling = vm
        for n in ("BertConfig", "BertModel", "BertForPreTrainingLossMask", "BertForSeq2SeqDecoder"):
            setattr(pkg, n, getattr(vm, n))
    return vm
