from .continuous_policy import *  # noqa: F401,F403
from .continuous_policy import (UniformPolicyContinuous, DetContPolicy, FixGuassianContPolicy,  # noqa: F401
                                GuassianContPolicyBase, GuassianContPolicy, GuassianContPolicyBasicBias)
from .discrete_policies import (UniformPolicyDiscrete, EpsilonGreedyDQNDiscretePolicy,  # noqa: F401
                                EpsilonGreedyQRDQNDiscretePolicy, BootstrappedDQNDiscretePolicy,
                                CategoricalDisPolicy)
from .distribution import TanhNormal, set_noise_mode, get_noise_mode  # noqa: F401
