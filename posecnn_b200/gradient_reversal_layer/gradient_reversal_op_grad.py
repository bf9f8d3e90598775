"""Gradient registration stub for lib/gradient_reversal_layer/gradient_reversal_op_grad.py (`ops.RegisterGradient("Gradientreversal")` in the
reference): importing it must succeed (`lib/networks/network.py:6-26`).  The reversal itself (-lambda * grad) is applied inside
train.Trainer's backward pass, so there is nothing to register — `gradient_reversal_op.gradient_reversal_grad` raises when called."""
try:
    from . import gradient_reversal_op  # noqa: F401
except ImportError:  # posecnn_b200/ itself on sys.path (reference-style imports)
    import gradient_reversal_layer.gradient_reversal_op as gradient_reversal_op  # noqa: F401
