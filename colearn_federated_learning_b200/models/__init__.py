"""Model families: FFNN / TestingRemote / Net (reference), MLP / WideMLP / ResNet-18 (BASELINE)."""
from .mlp import (FFNN, MLP, Autoencoder, FFNNCategory, MLPNet, MLPSpec, Net, TestingRemote, WideMLP,  # noqa: F401
                  AE_SPEC, FFNN_CAT_SPEC, FFNN_SPEC, MLP_SPEC, NET_SPEC, TESTING_REMOTE_SPEC, WIDE_MLP_SPEC)
from .resnet import ResNet18  # noqa: F401
from .registry import (MODEL_REGISTRY, DEFAULT_LOSS, build_model, register_model, load_plugins, model_spec, param_layout,  # noqa: F401
                       num_params, flatten_params, unflatten_params, alias_params_to_arena,
                       state_dict_from_flat)
