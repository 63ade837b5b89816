"""Entry point with the reference's command line (main_diffusion.py:13-28):

    python main_diffusion.py --config=configs/res64.py --mode={train,uncond_gen,cond_gen,eval_metrics,eval_likelihood,make_partial,partial_from_depth,fit_grids,export,uncond_gen_interp,eval_completion,edit,distill} [--config.a.b=value ...]

The reference parses this with absl + ml_collections.config_flags (lock_config=False: overrides may create keys);
neither ml_collections nor network access is available here, so the same syntax is parsed directly.
Under `torchrun --nproc-per-node N` every rank drives its own GPU (LOCAL_RANK) and its own batch shard.
"""
import importlib.util
import logging
import os
import sys

import torch

from meshdiffusion_b200.compat.config_dict import parse_override_value
from meshdiffusion_b200.compat.install import ensure_ml_collections

MODES = ("train", "uncond_gen", "cond_gen", "eval_metrics", "eval_likelihood", "make_partial", "fit_grids", "export",
         "uncond_gen_interp", "eval_completion", "edit", "partial_from_depth", "distill")


def load_config_file(path):
    ensure_ml_collections()
    spec = importlib.util.spec_from_file_location("_mdb_config", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.get_config()


def parse_args(argv):
    config_path, mode, overrides = None, None, []
    it = iter(argv)
    for arg in it:
        if not arg.startswith("--"):
            raise SystemExit(f"Unexpected positional argument: {arg}")
        body = arg[2:]
        if "=" in body:
            key, value = body.split("=", 1)
        else:
            key, value = body, next(it, None)
            if value is None:
                raise SystemExit(f"Flag --{key} needs a value")
        if key == "config":
            config_path = value
        elif key == "mode":
            mode = value
        elif key.startswith("config."):
            overrides.append((key[len("config."):], parse_override_value(value)))
        else:
            raise SystemExit(f"Unknown command line flag '{key}'")
    if config_path is None:
        raise SystemExit("Flag --config must have a value other than None.")
    if mode not in MODES:
        raise SystemExit(f"Flag --mode must be one of {MODES}")
    return config_path, mode, overrides


def main(argv=None):
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(message)s")
    config_path, mode, overrides = parse_args(sys.argv[1:] if argv is None else argv)
    config = load_config_file(config_path)
    for dotted, value in overrides:
        config.set_by_path(dotted, value)
    if torch.cuda.is_available():
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        config.device = torch.device(f"cuda:{local}")
    from meshdiffusion_b200.diffusion import evaler
    if mode == "train":
        from meshdiffusion_b200.diffusion import trainer
        trainer.train(config)
    elif mode == "uncond_gen":
        evaler.uncond_gen(config)
    elif mode == "cond_gen":
        evaler.cond_gen(config)
    elif mode == "eval_metrics":
        from meshdiffusion_b200.diffusion import gen_metrics
        gen_metrics.eval_metrics(config)
    elif mode == "eval_likelihood":
        from meshdiffusion_b200.diffusion import eval_likelihood
        eval_likelihood.eval_likelihood(config)
    elif mode == "make_partial":
        evaler.make_partial(config)
    elif mode == "partial_from_depth":
        evaler.partial_from_depth(config)
    elif mode == "fit_grids":
        from meshdiffusion_b200.diffusion import fit_grids
        fit_grids.fit_grids(config)
    elif mode == "export":
        from meshdiffusion_b200.diffusion import export
        export.export(config)
    elif mode == "uncond_gen_interp":
        from meshdiffusion_b200.diffusion import interp
        interp.uncond_gen_interp(config)
    elif mode == "eval_completion":
        from meshdiffusion_b200.diffusion import completion
        completion.eval_completion(config)
    elif mode == "edit":
        from meshdiffusion_b200.diffusion import edit
        edit.edit(config)
    elif mode == "distill":
        from meshdiffusion_b200.diffusion import distill
        distill.distill(config)


if __name__ == "__main__":
    main()
