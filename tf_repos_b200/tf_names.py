"""TF-checkpoint naming (SURVEY.md 8f-4).  `model.variables()` already uses the reference graph's variable names
(`fm_bias`, `fm_w`, `fm_v`, `Deep-part/mlp0/weights`, ...: DeepFM.py:114-116,156,165); this module adds the names
tf.train.Saver gives the OPTIMIZER state, so a whole training state can travel as one `{tf name: array}` mapping:

    Adam      <var>/Adam (m), <var>/Adam_1 (v), beta1_power, beta2_power      [TF-sem: slot names "m"/"v" are saved as
    Adagrad   <var>/Adagrad                                                     Adam / Adam_1 by Optimizer._slot_dict order]
    Momentum  <var>/Momentum
    Ftrl      <var>/Ftrl (accum), <var>/Ftrl_1 (linear)
    global_step

`tf_tensors` is the one place that decides which model tensor carries which name; `state_dict_tf`, `load_state_dict_tf`
and the TensorFlow checkpoint bundles of tf_checkpoint.py all iterate it.
`export_npz` / `import_npz` write/read that mapping as a NumPy archive ("/" kept in the keys).  On the TensorFlow side
`tf.train.load_checkpoint(path).get_tensor(name)` produces, and `tf.assign` / `init_from_checkpoint` consumes, exactly
these names and shapes (INTEGRATION.md section 6).
"""
from __future__ import annotations

from typing import Dict, Iterator, Tuple

import numpy as np
import torch

SLOT_SUFFIX = {"Adam": ["Adam", "Adam_1"], "Adagrad": ["Adagrad"], "Momentum": ["Momentum"], "ftrl": ["Ftrl", "Ftrl_1"]}


def tf_tensors(model, optimizer: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
    """(TF checkpoint name, tensor) for every tensor of a training state, in one order: the model's variables, the
    table slots, the dense slots (views into the flat slot buffers), `beta1_power` / `beta2_power` (0-d views of the
    optimizer state) and `global_step`.  optimizer=False yields the variables and `global_step` only (what a PREDICT
    graph holds).  Every tensor is the model's own storage, written in place by a restore, except `global_step`: a
    fresh 0-d int64 tensor holding model.global_step, to be handed back to set_global_step() after it is written."""
    model.flush()
    yield from model.variables().items()
    if optimizer:
        suf = SLOT_SUFFIX[model.opt.name]
        for t in model.tables:
            for s, sfx in zip(t.slots, suf):
                yield f"{t.name}/{sfx}", s
        for k, sfx in enumerate(suf):
            flat = model.dense.slots[k]
            for name, view in model.dense.views.items():
                off = (view.data_ptr() - model.dense.flat.data_ptr()) // 4
                yield f"{name}/{sfx}", flat[off:off + view.numel()].view(view.shape)
        if model.opt.name == "Adam":
            yield "beta1_power", model.opt.state[0]
            yield "beta2_power", model.opt.state[1]
    yield "global_step", torch.tensor(model.global_step, dtype=torch.int64, device=model.opt.state.device)


def set_global_step(model, step: int):
    model.global_step = int(step)
    model.opt.state[3] = float(model.global_step)


def state_dict_tf(model) -> Dict[str, np.ndarray]:
    """{TF checkpoint name: array} for variables, optimizer slots, Adam beta powers and global_step."""
    out: Dict[str, np.ndarray] = {}
    for name, t in tf_tensors(model):
        a = t.detach().cpu().numpy().copy()
        out[name] = a[()] if a.ndim == 0 else a
    return out


def load_state_dict_tf(model, values: Dict[str, np.ndarray], strict: bool = True):
    pairs = list(tf_tensors(model))
    missing = [k for k, _ in pairs if k not in values] if strict else []
    if missing:
        raise KeyError(f"missing TF variables: {missing[:5]}{' ...' if len(missing) > 5 else ''}")
    for name, dst in pairs:
        if name not in values:
            continue
        if name == "global_step":
            set_global_step(model, int(values[name]))
        else:
            dst.copy_(torch.as_tensor(np.asarray(values[name]), dtype=torch.float32).to(dst.device).reshape(dst.shape))


def export_npz(model, path: str):
    np.savez(path, **{k.replace("/", "|"): v for k, v in state_dict_tf(model).items()})


def import_npz(model, path: str, strict: bool = True):
    with np.load(path) as z:
        load_state_dict_tf(model, {k.replace("|", "/"): z[k] for k in z.files}, strict)
