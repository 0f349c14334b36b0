"""`bench.py --impl reference --model bert --dtype bf16` (the default dtype for BERT, as BASELINE.json names the
config "BERT-large pretraining bf16"): the reference's DeAR path is fp32-only, so the same-precision baseline is the
reference's PyTorch-DDP recipe (baseline/_ref/pytorch-ddp/bert_benchmark.py:58-126: HF ``BertForPreTraining``,
``DistributedDataParallel`` over NCCL, SGD lr=2e-5, its synthetic batch, criterion and ``benchmark_step`` incl. the
``torch.cuda.synchronize()``) with the model cast to bf16 — BASELINE.md section 2.  ``--dtype fp32`` runs the
reference's DeAR optimizer below.

`bench.py --impl reference`: the reference's own DeAR optimizer (baseline/_ref/dear/dopt_rsag.py,
tensorfusion.py — unmodified) driven exactly as its benchmark driver does
(baseline/_ref/dear/imagenet_benchmark.py:73-136: torchvision model, SGD lr=0.01*size,
DistributedOptimizer iff size>1, broadcast_parameters, benchmark_step incl. its
torch.cuda.synchronize()), timed with the same protocol as the dear arm.
"""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")


def _unavailable(why):
    print(json.dumps({"impl": "reference", "unavailable": why}), flush=True)
    return 0


def run(args):
    if not os.path.isdir(os.path.join(REF, "dear")):
        src = os.environ.get("DEAR_REFERENCE_DIR", "")
        if src and os.path.isdir(os.path.join(src, "dear")):
            import shutil
            shutil.copytree(src, REF, dirs_exist_ok=True)
        else:
            return _unavailable("baseline/_ref is missing and DEAR_REFERENCE_DIR does not name a checkout of the reference "
                                "(the reference has no setup.py; comm_core needs MPI)")
    try:
        import torch
        if not torch.cuda.is_available():
            return _unavailable("the reference is CUDA-only (no CPU path)")
        import torchvision  # noqa: F401
    except Exception as exc:  # pragma: no cover
        return _unavailable("missing dependency: %r" % (exc,))

    sys.path.insert(0, os.path.join(REF, "dear"))
    sys.path.insert(0, HERE)                      # comm_core stand-in (NCCL via torch.distributed)
    import torch.backends.cudnn as cudnn
    import torch.nn.functional as F
    import torch.optim as optim
    from torchvision import models
    import comm_core
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank % torch.cuda.device_count())
    comm_core.init()
    import dopt_rsag as hvd                      # the reference module, unmodified

    hvd.init()
    cudnn.benchmark = True
    rank, world = hvd.rank(), hvd.size()
    is_bert = args.model in ("bert", "bert_large", "bert_base")
    bf16_ddp = is_bert and getattr(args, "dtype", "fp32") == "bf16"
    B = args.batch_size
    if is_bert:
        # dear/bert_benchmark.py:72-122, with the installed transformers (5.x returns ModelOutput, so
        # return_dict=False restores the tuple the reference unpacks)
        try:
            from transformers import BertConfig, BertForPreTraining
        except Exception as exc:
            return _unavailable("transformers is not importable: %r" % (exc,))
        cfg_file = "bert_base_config.json" if args.model == "bert_base" else "bert_config.json"
        config = BertConfig.from_json_file(os.path.join(REF, "dear", cfg_file))
        if config.vocab_size % 8 != 0:
            config.vocab_size += 8 - (config.vocab_size % 8)
        vocab_size = config.vocab_size
        model = BertForPreTraining(config).cuda()
        if bf16_ddp:
            model = model.to(torch.bfloat16)
        max_len = args.sentence_len
        input_ids = (torch.rand(B, max_len) * 2000).long().cuda()
        attention_masks = torch.rand(B, max_len).long().cuda()
        token_type_ids = torch.rand(B, max_len).long().cuda()
        next_sentence_label = torch.rand(B, 1).long().cuda()
        masked_lm_labels = torch.rand(B, max_len).long().cuda()
        loss_fct = torch.nn.CrossEntropyLoss(ignore_index=-1)
        optimizer = optim.SGD(model.parameters(), lr=2e-5)
        size = max_len
        unit, metric = "samples/s", "samples/sec (BERT-%s pre-training, seq %d, DeAR tensor fusion)" % (
            "base" if args.model == "bert_base" else "large", max_len)
    else:
        if not hasattr(models, args.model):
            return _unavailable("model %s is not in torchvision" % args.model)
        model = getattr(models, args.model)().cuda()
        optimizer = optim.SGD(model.parameters(), lr=0.01 * world)
        size = 299 if args.model == "inception_v3" else 224
        data = torch.randn(B, 3, size, size).cuda()
        target = torch.LongTensor(B).random_() % 1000
        target = target.cuda()
        unit = "images/s"
        metric = "images/sec (ResNet-50 synthetic ImageNet training, DeAR tensor fusion)" if args.model == "resnet50" \
            else "images/sec (%s synthetic training, DeAR tensor fusion)" % args.model
    if bf16_ddp:
        if world > 1:       # pytorch-ddp/bert_benchmark.py:84 (DDP broadcasts the parameters itself)
            model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[torch.cuda.current_device()])
            optimizer = optim.SGD(model.parameters(), lr=2e-5)
    elif world > 1:
        optimizer = hvd.DistributedOptimizer(optimizer, model=model)
        hvd.broadcast_parameters(model.state_dict(), root_rank=0)

    if is_bert:
        def benchmark_step(ids=None, tgt=None):
            ids = input_ids if ids is None else ids
            optimizer.zero_grad()
            prediction_scores, seq_relationship_score = model(input_ids=ids, token_type_ids=token_type_ids,
                                                              attention_mask=attention_masks, return_dict=False)
            loss = loss_fct(prediction_scores.view(-1, vocab_size), masked_lm_labels.view(-1)) + \
                loss_fct(seq_relationship_score.view(-1, 2), next_sentence_label.view(-1))
            loss.backward()
            optimizer.step()
            torch.cuda.synchronize()
            return loss
    else:
        def benchmark_step(d=None, t=None):
            d = data if d is None else d
            t = target if t is None else t
            optimizer.zero_grad()
            output = model(d)
            loss = F.cross_entropy(output, t)
            loss.backward()
            optimizer.step()
            torch.cuda.synchronize()
            return loss

    import torch.distributed as dist

    def barrier():
        if world > 1:
            dist.barrier()

    for _ in range(args.warmup):
        benchmark_step()

    def timed(fn, n):
        barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize(); barrier()
        return e0.elapsed_time(e1)

    def maxr(v):
        if world == 1:
            return v
        t = torch.tensor([v], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    from dear_pytorch_b200.utils.clocks import ClockSampler   # nvidia-smi sampler only (not on the timed path)
    sampler = ClockSampler(torch.cuda.current_device()).start() if rank == 0 else None
    w0 = time.time()
    ms = maxr(timed(benchmark_step, args.steps))
    w1 = time.time()

    e2e = None
    if not args.no_e2e:
        if is_bert:
            hx = [(torch.rand(B, size) * 2000).long().pin_memory() for _ in range(4)]
            hy = [torch.zeros(1, dtype=torch.long).pin_memory() for _ in range(4)]
        else:
            hx = [torch.randn(B, 3, size, size).pin_memory() for _ in range(4)]
            hy = [(torch.LongTensor(B).random_() % 1000).pin_memory() for _ in range(4)]
        k = [0]
        losses = []

        def one():
            i = k[0] % 4
            k[0] += 1
            d = hx[i].cuda(non_blocking=True)
            t = hy[i].cuda(non_blocking=True)
            losses.append(benchmark_step(d, t).item())
        for _ in range(min(3, args.warmup)):
            one()
        ms_e = maxr(timed(one, args.steps))
        e2e = {"value": round(B * world * args.steps / (ms_e / 1e3), 2), "unit": unit,
               "h2d_bytes_per_step": int(hx[0].numel() * hx[0].element_size() + hy[0].numel() * 8), "d2h_bytes_per_step": 4,
               "ms_per_step": round(ms_e / args.steps, 4)}
    clocks = None
    if sampler is not None:
        sampler.stop()
        clocks = sampler.summary(w0, w1)
    if rank == 0:
        value = B * world * args.steps / (ms / 1e3)
        print(json.dumps({
            "metric": metric, "value": round(value, 2),
            "unit": unit, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": round(ms / args.steps, 4), "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16" if bf16_ddp else ("fp32" if is_bert else "fp32 (TF32 convolutions, torch defaults)"),
            "data": "synthetic", "impl": "reference",
            "config": {"model": args.model, "global_batch": B * world, "batch_per_gpu": B, ("seq_len" if is_bert else "image"): size,
                       "parallelism": "dp%d" % world, "optimizer": "SGD",
                       "path": ("baseline/_ref/pytorch-ddp/bert_benchmark.py recipe (DistributedDataParallel over NCCL), model in bf16"
                                if bf16_ddp else
                                "baseline/_ref/dear/dopt_rsag.py over NCCL (comm_core stand-in: torch.distributed)"),
                       "l2": "no explicit flush: working set far larger than L2"},
            "e2e": e2e, "gpu_launches": 0, "clocks": clocks}), flush=True)
    if world > 1:
        dist.destroy_process_group()
    return 0
