"""update_experiment_path / print_args / save_args_to_yaml used by the harness (reference utils/project_utils.py)."""
import os

import yaml


def update_experiment_path(args, short=False):
    """Append an experiment directory named from the run's settings to ``args.output_path``, create it and return
    ``args``: ``[<exp_prefix>-]<train_architecture>[_<lora_rank>]``, followed unless ``short`` by
    ``_pose_cfg-<pose_cfg>_mouth_cfg-<mouth_cfg>_pose_relax-<pose_relax>-f<pose_relax_num>-<ft|scratch>`` (ft when
    ``pretrained_lora_path`` is set)."""
    mode = "ft" if args.pretrained_lora_path else "scratch"
    parts = [f"{args.train_architecture}"]
    if args.train_architecture == "lora":
        parts.append(f"{args.lora_rank}")
    if not short:
        parts += [f"pose_cfg-{args.pose_cfg}", f"mouth_cfg-{args.mouth_cfg}",
                  f"pose_relax-{args.pose_relax}-f{args.pose_relax_num}-{mode}"]
    name = "_".join(parts)
    if args.exp_prefix:
        name = f"{args.exp_prefix}-{name}"
    args.output_path = os.path.join(args.output_path, name)
    print(f"Experiment path: {args.output_path}")
    os.makedirs(args.output_path, exist_ok=True)
    return args


def print_args(args):
    d = vars(args)
    width = max(len(k) for k in d) if d else 0
    print("=" * 80)
    print("CONFIGURATION PARAMETERS:")
    print("=" * 80)
    for k in sorted(d):
        print(f"  {k.ljust(width)} : {d[k]}")
    print("=" * 80)
    print(f"Total number of cfg parameters: {len(d)}")
    print("=" * 80)


def save_args_to_yaml(args, output_path):
    """rank-0 only, like the reference (:47-109)."""
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
            return
    except Exception:  # noqa: BLE001
        pass
    os.makedirs(output_path, exist_ok=True)
    with open(os.path.join(output_path, "args.yaml"), "w") as f:
        yaml.safe_dump({k: (v if isinstance(v, (int, float, str, bool, list, type(None))) else str(v))
                        for k, v in vars(args).items()}, f, sort_keys=True)
