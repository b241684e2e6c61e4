"""Layer-decay parameter groups and the optimizer factory of the fine-tuning scripts, as the tests need them:

- a parameter's layer is 0 for the global / class / mask tokens, the position table and the input adapters, i + 1 for
  encoder block i, and the last layer for everything else (the heads);
- it takes no weight decay when it is 1-D, a bias or listed in the skip list;
- one group per (layer, decay or not), in order of first appearance, with {"weight_decay", "params", "lr_scale"};
- create_optimizer builds `optim.AdamW(groups, lr=..., weight_decay=0.)` (or over all parameters with the weight decay
  when there is none to filter), `optim` being this module's global."""
from torch import optim as optim  # noqa: F401  (rebound by the overlay under MMAE_FLAT_ADAMW=1)

_LAYER_ZERO_NAMES = ("cls_token", "mask_token", "pos_embed", "global_tokens")


def get_num_layer_for_vit(var_name, num_max_layer):
    if var_name in _LAYER_ZERO_NAMES or var_name.startswith(("patch_embed", "input_adapters")):
        return 0
    if var_name.startswith(("blocks", "encoder")):
        return int(var_name.split(".")[1]) + 1
    return num_max_layer - 1


class LayerDecayValueAssigner:
    def __init__(self, values):
        self.values = values

    def get_scale(self, layer_id):
        return self.values[layer_id]

    def get_layer_id(self, var_name):
        return get_num_layer_for_vit(var_name, len(self.values))


def get_parameter_groups(model, weight_decay=1e-5, skip_list=(), get_num_layer=None, get_layer_scale=None):
    groups = {}
    for name, param in model.named_parameters():
        if not param.requires_grad:
            continue
        no_decay = param.ndim == 1 or name.endswith(".bias") or name in skip_list
        key = "no_decay" if no_decay else "decay"
        layer = None
        if get_num_layer is not None:
            layer = get_num_layer(name)
            key = "layer_%d_%s" % (layer, key)
        if key not in groups:
            scale = get_layer_scale(layer) if get_layer_scale is not None else 1.0
            groups[key] = {"weight_decay": 0.0 if no_decay else weight_decay, "params": [], "lr_scale": scale}
        groups[key]["params"].append(param)
    return list(groups.values())


def create_optimizer(args, model, get_num_layer=None, get_layer_scale=None, filter_bias_and_bn=True, skip_list=None):
    weight_decay = args.weight_decay
    if isinstance(model, dict):          # pre-training: the model and the task balancer
        parameters = [{"params": [p for p in model["model"].parameters() if p.requires_grad], "lr_scale": 1.0},
                      {"params": [p for p in model["balancer"].parameters() if p.requires_grad],
                       "lr_scale": args.balancer_lr_scale}]
    elif weight_decay and filter_bias_and_bn:
        skip = skip_list if skip_list is not None else (model.no_weight_decay() if hasattr(model, "no_weight_decay")
                                                        else {})
        parameters = get_parameter_groups(model, weight_decay, skip, get_num_layer, get_layer_scale)
        weight_decay = 0.0
    else:
        parameters = model.parameters()
    opt_args = dict(lr=args.lr, weight_decay=weight_decay)
    if getattr(args, "opt_eps", None) is not None:
        opt_args["eps"] = args.opt_eps
    if getattr(args, "opt_betas", None) is not None:
        opt_args["betas"] = args.opt_betas
    name = args.opt.lower().split("_")[-1]
    if name in ("sgd", "nesterov", "momentum"):
        opt_args.pop("eps", None)
        return optim.SGD(parameters, momentum=args.momentum, nesterov=name != "momentum", **opt_args)
    if name == "adam":
        return optim.Adam(parameters, **opt_args)
    if name == "adamw":
        return optim.AdamW(parameters, **opt_args)
    raise ValueError("Invalid optimizer %r" % args.opt)


def layer_decay_assigner(model, layer_decay):
    """run_finetuning_cls.py's LayerDecayValueAssigner for `model` (one value per layer, the heads' last)."""
    num_layers = model.get_num_layers()
    return LayerDecayValueAssigner([layer_decay ** (num_layers + 1 - i) for i in range(num_layers + 2)])

