"""Gradientreversal — import stub for lib/gradient_reversal_layer/gradient_reversal_op.py:1-7.

`lib/networks/network.py:6-26` imports this module unconditionally, so it must exist for the reference's network code
to import against this package (SURVEY.md §8(b): "stub modules for the other ops").  The reference network calls the op
under adaptation=True (vgg16_convs.py:207: identity forward, -lambda * grad backward).  posecnn_b200 implements that
reversal inside the training step instead of as a standalone op: Trainer multiplies the domain branch's pool_score
gradient by -lambda where it merges it with the pose head's (pcnn_domain_grad_merge, DESIGN.md §10).  The symbols exist,
calling them fails loudly; there is no CPU or library fallback.
"""
from __future__ import annotations


def _out_of_scope(name):
    def op(*args, **kwargs):
        raise NotImplementedError("%s (%s) is not provided as a standalone op: posecnn_b200 applies the gradient reversal of "
                                  "vgg16_convs(adaptation=True) inside train.Trainer's backward pass" % (name, "Gradientreversal"))
    op.__name__ = name
    return op


gradient_reversal = _out_of_scope("gradient_reversal")
gradient_reversal_grad = _out_of_scope("gradient_reversal_grad")
