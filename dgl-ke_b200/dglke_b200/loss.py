"""LossGenerator (reference: models/pytorch/loss.py:41-98, models/base_loss.py) over kge_loss_grad.

All four criteria of the reference (Hinge, Logistic, Logsigmoid, BCE: loss.py:10-38), the self-adversarial negative
weighting, edge-importance weights and the pairwise form (loss.py:76-80) run in the library (k_loss; the Logsigmoid family
without -pw also inside the fused wgmma kernel).  Logistic and BCE are the Logsigmoid criterion written differently and
share its kernels; the same argument errors as the reference's are raised (loss.py:58-62, base_loss.py:83-84)."""
import torch as th

from . import engine as E


class LazyLog(dict):
    """log dict {'pos_loss','neg_loss','loss','regularization'} whose floats are read from the device
    only when somebody looks (the reference pays 3-4 .item() syncs per step, tensor_models.py:55)."""
    KEYS = ("pos_loss", "neg_loss", "loss", "regularization")

    def __init__(self, log4, has_reg=True, lazy=False, only_loss=False):
        """only_loss: the pairwise form logs 'loss' alone (loss.py:78-80)"""
        super().__init__()
        # lazy: the scalars are written by a kernel that has not been enqueued yet (fused step: the update kernel
        # reduces them); an event recorded right after that kernel would be ideal, reading on first use after the
        # caller's update() is what the train loop does
        self._log4 = log4 if lazy else log4.clone()
        self._keys = self.KEYS if has_reg else self.KEYS[:3]
        if only_loss:
            self._keys = tuple(k for k in self._keys if k in ("loss", "regularization"))
        self._vals = None

    def _load(self):
        if self._vals is None:
            v = self._log4.cpu().tolist()
            self._vals = dict(zip(self.KEYS, v))
            for k in self._keys:
                dict.__setitem__(self, k, self._vals[k])
        return self._vals

    def __getitem__(self, k):
        self._load()
        return dict.__getitem__(self, k)

    def keys(self):
        return list(self._keys)

    def items(self):
        self._load()
        return dict.items(self)

    def __iter__(self):
        return iter(self._keys)

    def __len__(self):
        return len(self._keys)

    def __contains__(self, k):
        return k in self._keys


class FusedLoss:
    """What KEModel.forward returns as `loss`: the fused step has already produced every gradient,
    so backward() has nothing left to do (train_pytorch.py:145 keeps working unchanged)."""

    def __init__(self, log4, with_reg, lazy=False):
        self._log4, self._with_reg = log4, with_reg

    def backward(self):
        return None

    def item(self):
        v = self._log4.cpu().tolist()
        return v[2] + (v[3] if self._with_reg else 0.0)

    def detach(self):
        return self

    def __float__(self):
        return self.item()


class LossGenerator:
    def __init__(self, args, loss_genre="Logsigmoid", neg_adversarial_sampling=False, adversarial_temperature=1.0,
                 pairwise=False):
        if pairwise and neg_adversarial_sampling:
            raise ValueError("loss cannot be pairwise and adversarial sampled")                 # base_loss.py:83-84
        if loss_genre not in ("Hinge", "Logistic", "Logsigmoid", "BCE"):
            raise ValueError("loss genre %s is not support" % loss_genre)                       # loss.py:58-59
        if pairwise and loss_genre not in ("Logistic", "Hinge"):
            raise ValueError("{} loss cannot be applied to pairwise loss function".format(loss_genre))   # loss.py:61-62
        self.loss_genre = loss_genre
        self.margin = float(getattr(args, "margin", 1.0)) if args is not None else 1.0
        self.pairwise = bool(pairwise)
        self.neg_adversarial_sampling = bool(neg_adversarial_sampling)
        self.adversarial_temperature = adversarial_temperature if neg_adversarial_sampling else 0
        self.neg_label = 0 if loss_genre == "BCE" else -1

    def _hyper(self):
        return E.Hyper(model="DistMult", hidden_dim=4, adversarial=self.neg_adversarial_sampling,
                       adv_temperature=float(self.adversarial_temperature or 1.0), loss_genre=self.loss_genre,
                       margin=self.margin, pairwise=self.pairwise)

    def get_total_loss(self, pos_score, neg_score, edge_weight=None):
        """-> (loss 0-dim tensor, log).  Forward-only stand-alone op; d loss / d score is available
        through score_gradients()."""
        log4, _, _ = E.loss_grad(self._hyper(), pos_score, neg_score, edge_weight)
        log = LazyLog(log4, has_reg=False, only_loss=self.pairwise)
        return log4[2], log

    def score_gradients(self, pos_score, neg_score, edge_weight=None):
        _, dpos, dneg = E.loss_grad(self._hyper(), pos_score, neg_score, edge_weight)
        return dpos, dneg
