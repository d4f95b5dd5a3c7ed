"""B200-native drop-in for the one hot path of travistangvh/time-series-kafka-demo:
``output = model(x_arr, a_arr)`` (bin/predictStream.py:157) -> ``MyCNN.forward``
(bin/models.py:22-36), as hand-written sm_90a CUDA behind the C ABI in ``include/b2cnn.h``.

    from tskd_b200 import B200MyCNN, load_reference_checkpoint
    model = B200MyCNN.from_reference(load_reference_checkpoint("model/MyCNN5.pth")).eval()
    logit = model(x, age)                    # same call as the reference
    prob  = model.predict(windows, ages)     # batched, one independent window per row
    loss  = B200Trainer(model).step(x, age, target)   # one training step (bin/utils.py:200-208) on the device
    model = B200TrainableMyCNN.from_reference(sd).cuda().train()   # torch autograd + any loss / optimizer
    scorer = SlidingScorer(model, n_patients, stride)   # sliding windows: one push of new samples per trigger

There is no CPU fallback: constructing a model without the CUDA library or a GPU raises.
"""
from .arch import ArchConfig, ARCH_PRESETS, arch_from_state_dict  # noqa: F401
from .capi import LibraryNotBuilt, lib_path, load_library  # noqa: F401
from .checkpoint import load_reference_checkpoint  # noqa: F401
from .model import B200MyCNN  # noqa: F401
from .trainer import B200HeadTrainer, B200Trainer  # noqa: F401
from .autograd import B200TrainableMyCNN, mycnn_train_forward, mycnn_train_record_forward  # noqa: F401
from .slide import SlidingScorer  # noqa: F401
from .stream import PatientRing  # noqa: F401
from . import synth  # noqa: F401

__all__ = ["ArchConfig", "ARCH_PRESETS", "arch_from_state_dict", "B200MyCNN", "B200Trainer", "B200HeadTrainer", "B200TrainableMyCNN", "mycnn_train_forward", "mycnn_train_record_forward", "SlidingScorer", "PatientRing",
           "load_reference_checkpoint", "load_library", "lib_path", "LibraryNotBuilt", "synth"]
