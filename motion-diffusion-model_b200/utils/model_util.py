"""Factory: args -> (model, diffusion); checkpoint loading (host mirror of the reference's utils/model_util.py)."""
import torch

from ..diffusion import gaussian_diffusion as gd
from ..diffusion.respace import SpacedDiffusion, space_timesteps
from ..model.mdm import MDM

HML_EE_JOINT_NAMES = ["left_foot", "right_foot", "left_wrist", "right_wrist", "head"]  # data_loaders/humanml_utils.py


def get_cond_mode(args):
    """reference utils/parser_util.py:269-276."""
    if getattr(args, "unconstrained", False):
        return "no_cond"
    if args.dataset in ["kit", "humanml"]:
        return "text"
    return "action"


def get_model_args(args, data):
    """reference utils/model_util.py:24-71."""
    num_actions = getattr(getattr(data, "dataset", None), "num_actions", 1)
    data_rep, njoints, nfeats, goal_names = "rot6d", 25, 6, []
    if args.dataset == "humanml":
        data_rep, njoints, nfeats = "hml_vec", 263, 1
        goal_names = ["pelvis"] + HML_EE_JOINT_NAMES
    elif args.dataset == "kit":
        data_rep, njoints, nfeats = "hml_vec", 251, 1
    if not hasattr(args, "pred_len"):
        args.pred_len = 0
        args.context_len = 0
    extra = args.__dict__
    return {
        "modeltype": "", "njoints": njoints, "nfeats": nfeats, "num_actions": num_actions, "translation": True,
        "pose_rep": "rot6d", "glob": True, "glob_rot": True, "latent_dim": args.latent_dim, "ff_size": 1024,
        "num_layers": args.layers, "num_heads": 4, "dropout": 0.1, "activation": "gelu", "data_rep": data_rep,
        "cond_mode": get_cond_mode(args), "cond_mask_prob": args.cond_mask_prob, "action_emb": "tensor",
        "arch": args.arch, "emb_trans_dec": args.emb_trans_dec, "clip_version": "ViT-B/32", "dataset": args.dataset,
        # an args.json written before the BERT option has no text_encoder_type: the reference then loads CLIP
        "text_encoder_type": extra.get("text_encoder_type", "clip"), "pos_embed_max_len": args.pos_embed_max_len,
        "mask_frames": args.mask_frames, "pred_len": args.pred_len, "context_len": args.context_len,
        "emb_policy": extra.get("emb_policy", "add"), "all_goal_joint_names": goal_names,
        # apply_rules (reference utils/parser_util.py:51-53): a target-location loss implies the target encoder
        "multi_target_cond": extra.get("multi_target_cond", False) or extra.get("lambda_target_loc", 0.0) > 0.0,
        "multi_encoder_type": extra.get("multi_encoder_type", "multi"),
        "target_enc_layers": extra.get("target_enc_layers", 1),
        # engine-only knob: how many model timesteps get a pre-computed timestep embedding
        "num_model_timesteps": max(1000, int(args.diffusion_steps)),
    }


def create_gaussian_diffusion(args):
    """reference utils/model_util.py:75-116: x0-prediction, fixed variance, identity respacing."""
    steps = args.diffusion_steps
    betas = gd.get_named_beta_schedule(args.noise_schedule, steps, 1.0)
    return SpacedDiffusion(
        use_timesteps=space_timesteps(steps, [steps]),
        betas=betas,
        model_mean_type=gd.ModelMeanType.START_X,
        model_var_type=gd.ModelVarType.FIXED_SMALL if args.sigma_small else gd.ModelVarType.FIXED_LARGE,
        loss_type=gd.LossType.MSE,
        rescale_timesteps=False,
        lambda_vel=args.lambda_vel,
        lambda_rcxyz=args.lambda_rcxyz,
        lambda_fc=args.lambda_fc,
        lambda_target_loc=getattr(args, "lambda_target_loc", 0.0),
    )


def create_model_and_diffusion(args, data):
    """reference utils/model_util.py:18-21."""
    return MDM(**get_model_args(args, data)), create_gaussian_diffusion(args)


def load_model_wo_clip(model, state_dict):
    """reference utils/model_util.py:8-15: the positional tables are recomputed, CLIP weights are not stored."""
    state_dict = dict(state_dict)
    state_dict.pop("sequence_pos_encoder.pe", None)
    state_dict.pop("embed_timestep.sequence_pos_encoder.pe", None)
    missing, unexpected = model.load_state_dict(state_dict, strict=False)
    assert len(unexpected) == 0, unexpected
    assert all(k.startswith("clip_model.") or "sequence_pos_encoder" in k for k in missing), missing


def load_saved_model(model, model_path, use_avg: bool = False):
    """reference utils/model_util.py:118-132 (EMA-aware checkpoint layouts)."""
    state_dict = torch.load(model_path, map_location="cpu")
    if use_avg and "model_avg" in state_dict:
        state_dict = state_dict["model_avg"]
    elif "model" in state_dict:
        state_dict = state_dict["model"]
    load_model_wo_clip(model, state_dict)
    return model
