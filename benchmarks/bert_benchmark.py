#!/usr/bin/env python
"""Synthetic BERT pre-training benchmark (counterpart of */bert_benchmark.py in the reference).

    torchrun --nproc-per-node 8 benchmarks/bert_benchmark.py --model bert --batch-size 32 --sentence-len 128 --dtype bf16
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: E402
from common import dear  # noqa: E402
from dear_pytorch_b200.models import bert as bert_models  # noqa: E402
from dear_pytorch_b200.utils.train import TrainStep  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description="DeAR synthetic BERT benchmark",
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    ap.add_argument("--model", type=str, default="bert", choices=["bert", "bert_large", "bert_base"])
    ap.add_argument("--sentence-len", type=int, default=128)
    ap.add_argument("--lr", type=float, default=2e-5)
    ap.add_argument("--config", type=str, default=None, help="optional JSON file with BertConfig fields")
    ap.add_argument("--fused-ln", type=int, default=1, help="dropout + add + LayerNorm in one kernel (CUDA)")
    ap.add_argument("--tc-ffn", type=int, default=0, help="feed-forward block on the wgmma GEMMs (CUDA, bf16; opt-in)")
    common.add_common_args(ap)
    args = ap.parse_args(argv)
    method, cuda = common.init_runtime(args)
    device = dear.device()
    dtype = args.dtype or ("bf16" if args.fp16 else "fp32")

    # architecture hyper-parameters: models/bert.py (BERT_LARGE = 24 layers / 1024 hidden / 16 heads / 4096 FFN,
    # BERT_BASE = 12 / 768 / 12 / 3072; vocabulary 30522) or a user-supplied JSON file
    if args.config:
        import json
        with open(args.config) as f:
            cfg = bert_models.BertConfig(**{k: v for k, v in json.load(f).items()
                                            if k in bert_models.BertConfig.__dataclass_fields__})
    else:
        cfg = bert_models.BERT_BASE if args.model == "bert_base" else bert_models.BERT_LARGE
    model = bert_models.BertForPreTraining(cfg, fused_ln=bool(args.fused_ln) and cuda,
                                           tc_ffn=bool(args.tc_ffn) and cuda and dtype == "bf16").to(device)
    # (vocabulary padded to a multiple of 8)
    if dtype == "bf16":
        model = model.to(torch.bfloat16)
    criterion = bert_models.BertPretrainingCriterion(model.vocab_size)
    ids, mask, types, nsp, mlm = bert_models.synthetic_batch(args.batch_size, args.sentence_len, model.vocab_size, device)

    optimizer = common.make_base_optimizer(args, model.parameters(), args.lr)

    def profile():
        from dear_pytorch_b200.utils.profiling import benchmark
        return benchmark(model, (ids, types, mask, (mlm, nsp)), criterion, task="bert", warmup=3, iters=10)
    model, optimizer = common.wrap_optimizer(method, args, model, optimizer, profile)
    if dear.size() > 1 and method != "single":
        dear.broadcast_parameters(model.state_dict(), root_rank=0)

    def loss_fn(out, target):
        return criterion(out[0], out[1], target[0], target[1])
    step = TrainStep(model, optimizer, loss_fn, autocast_dtype=torch.bfloat16 if dtype == "amp" else None,
                     use_graph=bool(args.graph) and cuda)

    def sync(host=True):
        if hasattr(optimizer, "_dear"):
            optimizer._dear.synchronize(host=host)
        elif method in ("dear-rb", "bytescheduler") and hasattr(optimizer, "synchronize"):
            optimizer.synchronize()            # bytescheduler: deferred per-layer updates + its scheduler thread
        if cuda and host:
            torch.cuda.synchronize()

    common.log("BERT %s Pretraining, Sentence len: %d" % ("Base" if args.model == "bert_base" else "Large", args.sentence_len))
    common.log("Method: %s, dtype: %s, backend: %s" % (method, dtype, dear.backend()))
    common.log("Batch size: %d" % args.batch_size)
    res = common.run_timing(lambda: step(ids, types, mask, (mlm, nsp)), args, "sentences", args.batch_size, sync)
    common.finish(args, res, {"model": args.model, "method": method, "dtype": dtype, "world": dear.size(),
                              "batch_size": args.batch_size, "sentence_len": args.sentence_len})
    dear.shutdown()
    return res


if __name__ == "__main__":
    main()
