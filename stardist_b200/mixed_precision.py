"""Keras' mixed-precision policy for training: tf.keras.mixed_precision.Policy / set_global_policy / global_policy.

'float32' (the default) trains as before.  Under 'mixed_bfloat16' a UNetTrainer (and so train()) keeps fp32 parameters, Adam
state and loss, and runs every convolution, the heads and the class head on the bf16 tensor cores with bf16 activations and
bf16 gradients between layers (csrc/unet_train_bf16.cu, DESIGN.md 4.2).  bf16 has fp32's exponent range, so no loss scaling
is needed.  A trainer reads the policy once, when it is constructed.

Deliberate difference from Keras: prediction (predict*, optimize_thresholds and everything outside the trainer) ignores the
policy and always runs the fp32 executors; a model trained under 'mixed_bfloat16' saves fp32 weights and predicts exactly
like any other model.
"""

_NAMES = {'float32': ('float32', 'float32'), 'mixed_bfloat16': ('bfloat16', 'float32')}


class Policy:
    """a dtype policy: .name, .compute_dtype (the dtype layers compute in) and .variable_dtype (the dtype of the weights)"""

    def __init__(self, name):
        if isinstance(name, Policy):
            name = name.name
        if name == 'mixed_float16':
            raise NotImplementedError("policy 'mixed_float16' is not supported: float16 training needs loss scaling; "
                                      "use 'mixed_bfloat16', whose exponent range is float32's")
        if not isinstance(name, str) or name not in _NAMES:
            raise ValueError("Cannot convert value %r to a mixed precision Policy. Supported policies: %s"
                             % (name, ", ".join(repr(n) for n in _NAMES)))
        self._name = name
        self._compute_dtype, self._variable_dtype = _NAMES[name]

    @property
    def name(self):
        return self._name

    @property
    def compute_dtype(self):
        return self._compute_dtype

    @property
    def variable_dtype(self):
        return self._variable_dtype

    def __eq__(self, other):
        return isinstance(other, Policy) and other.name == self.name

    def __hash__(self):
        return hash(self._name)

    def __repr__(self):
        return '<Policy "%s">' % self._name


_global_policy = Policy('float32')


def set_global_policy(policy):
    """set the policy of trainers constructed from now on: a Policy or one of the names 'float32', 'mixed_bfloat16'"""
    global _global_policy
    _global_policy = policy if isinstance(policy, Policy) else Policy(policy)


def global_policy():
    """the current global Policy ('float32' unless set_global_policy changed it)"""
    return _global_policy
