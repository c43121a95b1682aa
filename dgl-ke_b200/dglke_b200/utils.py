"""Flag surface and save helpers of dglke_train (reference: utils.py:27-58,199-297; train.py:40-60).
Every flag of the reference parses with the same name, type and default."""
import argparse
import json
import math
import os


def get_compatible_batch_size(batch_size, neg_sample_size):
    # utils.py:27-33: round the batch up to a multiple of the negative sample size
    if neg_sample_size < batch_size and batch_size % neg_sample_size != 0:
        old = batch_size
        batch_size = int(math.ceil(batch_size / neg_sample_size) * neg_sample_size)
        print("batch size ({}) is incompatible to the negative sample size ({}). Change the batch size to {}".format(
            old, neg_sample_size, batch_size))
    return batch_size


def save_model(args, model, emap_file=None, rmap_file=None):
    """<dataset>_<model>_{entity,relation}.npy + config.json, the layout dglke_eval / dglke_predict read
    (utils.py:35-49, docs/source/format_out.rst)."""
    os.makedirs(args.save_path, exist_ok=True)
    print("Save model to {}".format(args.save_path))
    model.save_emb(args.save_path, args.dataset)
    save_config(args, emap_file, rmap_file)


def save_config(args, emap_file=None, rmap_file=None):
    """config.json of a checkpoint: the parsed arguments and the mapping files (utils.py:35-49)."""
    conf = dict(vars(args))
    conf.update({"emp_file": emap_file, "rmap_file": rmap_file})
    with open(os.path.join(args.save_path, "config.json"), "w") as f:
        json.dump(conf, f, indent=4)


def prepare_save_path(args):
    os.makedirs(args.save_path, exist_ok=True)
    folder = "{}_{}_".format(args.model_name, args.dataset)
    n = len([x for x in os.listdir(args.save_path) if x.startswith(folder)])
    args.save_path = os.path.join(args.save_path, folder + str(n))
    os.makedirs(args.save_path, exist_ok=True)


class CommonArgParser(argparse.ArgumentParser):
    def __init__(self):
        super(CommonArgParser, self).__init__()
        A = self.add_argument
        A("--model_name", default="TransE", choices=["TransE", "TransE_l1", "TransE_l2", "TransR", "RESCAL", "DistMult",
                                                      "ComplEx", "RotatE", "SimplE"], help="KGE model")
        A("--data_path", type=str, default="data", help="directory of the knowledge graph data")
        A("--dataset", type=str, default="FB15k", help="dataset name (prefix of the saved embeddings)")
        A("--format", type=str, default="built_in", help="built_in | raw_udd_{htr} | udd_{htr}")
        A("--data_files", type=str, default=None, nargs="+", help="[entity_file relation_file] train [valid] [test]")
        A("--delimiter", type=str, default="\t", help="column delimiter of the data files")
        A("--save_path", type=str, default="ckpts", help="where models and logs are saved")
        A("--no_save_emb", action="store_true", help="do not save the embeddings")
        A("--max_step", type=int, default=80000, help="number of training steps (batches)")
        A("--batch_size", type=int, default=1024, help="training batch size")
        A("--batch_size_eval", type=int, default=8, help="batch size for validation / test")
        A("--neg_sample_size", type=int, default=256, help="negatives per positive in training")
        A("--neg_deg_sample", action="store_true", help="degree-proportional negatives in training")
        A("--neg_deg_sample_eval", action="store_true", help="degree-proportional negatives in evaluation")
        A("--neg_sample_size_eval", type=int, default=-1, help="negatives per positive in evaluation")
        A("--eval_percent", type=float, default=1, help="fraction of edges sampled for evaluation")
        A("--no_eval_filter", action="store_true", help="do not filter true positives among the negatives")
        A("-log", "--log_interval", type=int, default=1000, help="print timers every x steps")
        A("--eval_interval", type=int, default=10000, help="validate every x steps")
        A("--test", action="store_true", help="evaluate on the test set after training")
        A("--num_proc", type=int, default=1, help="training processes (one per GPU here)")
        A("--num_thread", type=int, default=1, help="CPU threads per process")
        A("--force_sync_interval", type=int, default=-1, help="barrier between processes every x steps")
        A("--hidden_dim", type=int, default=400, help="embedding size")
        A("--lr", type=float, default=0.01, help="Adagrad learning rate")
        A("-g", "--gamma", type=float, default=12.0, help="margin of TransX / RotatE")
        A("-de", "--double_ent", action="store_true", help="double entity dim (RotatE, SimplE)")
        A("-dr", "--double_rel", action="store_true", help="double relation dim")
        A("-adv", "--neg_adversarial_sampling", action="store_true", help="self-adversarial negative weighting")
        A("-a", "--adversarial_temperature", default=1.0, type=float, help="temperature of -adv")
        A("-rc", "--regularization_coef", type=float, default=0.000002, help="regularization coefficient")
        A("-rn", "--regularization_norm", type=int, default=3, help="regularization norm")
        A("-pw", "--pairwise", action="store_true", help="pairwise loss")
        A("--loss_genre", default="Logsigmoid", choices=["Hinge", "Logistic", "Logsigmoid", "BCE"], help="loss")
        A("-m", "--margin", type=float, default=1.0, help="hinge margin")


class ArgParser(CommonArgParser):
    """train.py:40-60"""

    def __init__(self):
        super(ArgParser, self).__init__()
        A = self.add_argument
        A("--gpu", type=int, default=[-1], nargs="+", help="gpu ids, e.g. 0 1 2 4")
        A("--mix_cpu_gpu", action="store_true", help="(reference: table in host RAM) here: shard the table over the GPUs")
        A("--valid", action="store_true", help="validate during training")
        A("--rel_part", action="store_true", help="relation partitioning (not needed: relations are replicated)")
        A("--async_update", action="store_true", help="asynchronous entity update (always stream-async here)")
        A("--has_edge_importance", action="store_true", help="edges carry an importance weight")
        A("--host_sampler", action="store_true", help="(this package only) sample on the host with numpy instead of on the GPU")
