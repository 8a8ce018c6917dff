"""``parl.Model`` on PyTorch — host-side mirror of parl/core/torch/model.py:24-134.

Parameters stay torch tensors (on the H100); ``get_weights`` / ``set_weights`` keep the
reference's numpy-dict contract (one entry per ``state_dict`` key, in order) and
``sync_weights_to`` keeps ``target = decay*target + (1-decay)*self``
(behaviours pinned by parl/core/torch/tests/model_base_test_torch.py:53-335).
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

__all__ = ['Model']


class Model(nn.Module):
    def sync_weights_to(self, target_model, decay=0.0):
        assert target_model is not self, "cannot copy between identical model"
        assert isinstance(target_model, Model)
        assert self.__class__.__name__ == target_model.__class__.__name__, \
            "must be the same class for params syncing!"
        assert 0 <= decay <= 1
        targets = dict(target_model.named_parameters())
        with torch.no_grad():
            for name, src in self.named_parameters():
                dst = targets[name]
                # same three roundings as the reference expression (model.py:110-112): two products, one sum
                dst.copy_(decay * dst + (1 - decay) * src.detach().to(dst.device))

    def get_weights(self):
        # an OrderedDict in state_dict order, like the reference (model.py:115-123 fills state_dict() in place)
        return OrderedDict((k, v.detach().cpu().numpy()) for k, v in self.state_dict().items())

    def set_weights(self, weights):
        # like the reference (model.py:126-134): anything without .keys() fails with AttributeError, a wrong
        # shape with load_state_dict's RuntimeError
        self.load_state_dict({k: torch.from_numpy(np.asarray(weights[k])) for k in weights.keys()})
