"""ORACLE SUPPORT — imports the UNMODIFIED reference modules from the checkout at $VLP_REFERENCE_ROOT (golden-data generation only).

`import pytorch_pretrained_bert` fails on a modern stack: file_utils.py:20-21 needs boto3/botocore,
__init__.py:5-6 pulls optimization.py (torch._six, removed in torch 2) and optimization_fp16.py (apex).
Work-around that leaves the reference untouched (SURVEY.md §8c / Appendix A): stub the absent third-party
modules, register an empty package object whose __path__ points at the reference directory (so its
__init__ is bypassed) and import pytorch_pretrained_bert.modeling.  Without apex the reference falls back to
its own pure-PyTorch BertLayerNorm (modeling.py:179-192) — that is the arithmetic being pinned.

Never imported by the product or the tests: the tests compare with what oracle/make_golden.py stored under tests/golden/.
"""
import os
import pickle
import sys
import tempfile
import types

REF_ROOT = os.environ.get("VLP_REFERENCE_ROOT", "")


def available():
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "pytorch_pretrained_bert"))


def import_reference_modeling():
    if not available():
        raise RuntimeError(f"reference checkout not found (set VLP_REFERENCE_ROOT; got {REF_ROOT!r})")
    for name in ("boto3", "botocore", "botocore.exceptions"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["botocore.exceptions"].ClientError = Exception
    if "pytorch_pretrained_bert" not in sys.modules or not hasattr(sys.modules["pytorch_pretrained_bert"], "__path__"):
        pkg = types.ModuleType("pytorch_pretrained_bert")
        pkg.__path__ = [os.path.join(REF_ROOT, "pytorch_pretrained_bert")]
        sys.modules["pytorch_pretrained_bert"] = pkg
    import pytorch_pretrained_bert.modeling as m  # noqa: E402
    return m


def import_reference_optimization():
    """pytorch_pretrained_bert/optimization.py (BertAdam).  Its only obstacle on a modern stack is `from torch._six import
    container_abcs` (:27, unused by BertAdam itself): a stub module provides the name."""
    import collections.abc
    import_reference_modeling()          # registers the package object
    six = types.ModuleType("torch._six")
    six.container_abcs = collections.abc
    sys.modules.setdefault("torch._six", six)
    import pytorch_pretrained_bert.optimization as o  # noqa: E402
    return o


def build_reference_model(dims, state_dict, tasks="img2txt", decoder=False, **decoder_kw):
    """Instantiate the reference's BertForPreTrainingLossMask / BertForSeq2SeqDecoder (enable_butd=True) and
    load `state_dict`.  modeling.py:1008-1014 reads detectron_weights/fc7_{w,b}.pkl from the CWD at
    construction time; synthetic pickles are provided in a scratch directory and overwritten by the load."""
    import numpy as np
    import torch

    m = import_reference_modeling()
    cfg = m.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                       intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                       hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "detectron_weights"))
        pickle.dump(np.zeros((2048, 2048), np.float32), open(os.path.join(tmp, "detectron_weights", "fc7_w.pkl"), "wb"))
        pickle.dump(np.zeros((2048,), np.float32), open(os.path.join(tmp, "detectron_weights", "fc7_b.pkl"), "wb"))
        os.chdir(tmp)
        try:
            torch.manual_seed(0)
            if decoder:
                model = m.BertForSeq2SeqDecoder(cfg, enable_butd=True, len_vis_input=dims.regions, **decoder_kw)
            else:
                model = m.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=dims.regions, tasks=tasks)
        finally:
            os.chdir(cwd)
    sd = {k: v.clone() for k, v in state_dict.items()}
    missing, unexpected = model.load_state_dict(sd, strict=False)
    if unexpected or missing:   # explicit raise: this module is also run under `python -O`
        raise RuntimeError(f"reference state_dict mismatch: missing={missing} unexpected={unexpected}")
    return model
