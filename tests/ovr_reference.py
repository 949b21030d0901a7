"""Float64 reference for KernelSHAP on the one-vs-rest head -- TEST INFRASTRUCTURE.

``multiclass_reference.MultiOutputReference`` with the head swapped: C = R >= 3 linear scores, ``s_c = sigmoid(z_c)``,
``p_c = s_c / sum_c' s_c'`` (scikit-learn's ``_predict_proba_lr``), then the same weighted background mean, link and
constrained WLS per output.  The sigmoids are formed from ``log sigmoid`` so that rows where every class is far below
zero keep their ratios instead of dividing 0 by 0."""
import numpy as np

from multiclass_reference import MultiOutputReference


def ovr_probabilities(score):
    """[..., C] scores -> [..., C] normalised sigmoids."""
    ls = -np.logaddexp(0.0, -score)                       # log sigmoid
    e = np.exp(ls - ls.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


class OvrReference(MultiOutputReference):
    """``W`` [C, D], ``b`` [C], ``background`` [N, D], ``groups`` list of column lists, ``weights`` [N] or None,
    ``link`` 'logit' / 'identity'."""

    def __init__(self, W, b, background, groups, weights=None, link="logit"):
        super().__init__(W, b, background, groups, weights, head="softmax", link=link)
        self.head = "ovr"

    def _outputs(self, score):
        return ovr_probabilities(score)
