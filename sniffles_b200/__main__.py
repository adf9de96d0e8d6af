"""`python -m sniffles_b200 ARGS`: the reference's command line (sniffles:64-148) for its three run modes -- calling a sample
(`-i sample.bam -v out.vcf [--snf out.snf]`, call.call_sample), force calling (`--genotype-vcf`, genotype.genotype_vcf) and combining
samples (`-i a.snf b.snf ... -v out.vcf` or `-i samples.tsv -v out.vcf`, combine_run.combine_snfs).  CRAM input is not run from here.

Calling a sample, or combining samples, on N GPUs is one process per GPU:

    torchrun --standalone --nproc-per-node N -m sniffles_b200 -i sample.bam -v out.vcf --gpus N
    torchrun --standalone --nproc-per-node N -m sniffles_b200 -i a.snf b.snf ... -v out.vcf --gpus N

Every rank runs its share of the tasks and rank 0 writes the files, which are those of `--gpus 1`.  Only rank 0 logs the run's INFO
lines; the other ranks log warnings and errors, prefixed with their rank."""
import datetime
import logging
import os
import sys

from . import call, combine_run, genotype
from .config import SnifflesConfig

# how long a rank waits in a collective: the ranks finish their tasks at different times and wait for the last one in the gather
RANK_TIMEOUT = datetime.timedelta(hours=12)


def _rank_logging(rank):
    """ranks above 0 log warnings and errors only, each line prefixed with the rank"""
    if rank == 0:
        return
    root = logging.getLogger()
    root.setLevel(logging.WARNING)
    for h in root.handlers:
        fmt = h.formatter._fmt if h.formatter is not None else logging.BASIC_FORMAT
        h.setFormatter(logging.Formatter(f"rank {rank}: {fmt}"))


def _launch_ranks(world, log, refusal, run, error):
    """one rank of a torchrun launch with WORLD_SIZE > 1: ranks above 0 log warnings only; the mode's `refusal`, else more processes on
    this node than visible GPUs, refuses the launch alike on every rank; otherwise run(device) runs on this rank's GPU inside a gloo
    process group, and an `error` it raises is logged as fatal.  Every rank returns the same code."""
    import torch
    rank, local = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    _rank_logging(rank)
    local_world, n_dev = int(os.environ.get("LOCAL_WORLD_SIZE", world)), torch.cuda.device_count()
    if refusal is None and local_world > n_dev:           # LOCAL_RANK < device count on every rank of this node
        refusal = f"{local_world} processes on this node, but {n_dev} visible GPU(s): run one process per GPU"
    if refusal is not None:
        log.error(f"{refusal} (Fatal error, exiting.)")
        return 1
    import torch.distributed as tdist
    torch.cuda.set_device(local)
    tdist.init_process_group("gloo", timeout=RANK_TIMEOUT)
    try:
        run(local)
        code = 0
    except error as e:
        log.error(f"{e} (Fatal error, exiting.)")
        code = 1
    finally:
        tdist.destroy_process_group()
    return code


def _mismatch(config, world):
    return f"--gpus {config.gpus} does not match the {world} processes torchrun started (--nproc-per-node)"


def _main_ranks(config, world, log):
    """one rank of a torchrun launch of call mode with WORLD_SIZE > 1"""
    refusal = None
    if config.mode != "call_sample":
        refusal = f"--genotype-vcf runs on one GPU: run it without torchrun ({world} ranks would each write {config.vcf})"
    elif config.gpus != world:
        refusal = _mismatch(config, world)
    return _launch_ranks(world, log, refusal, lambda device: call.call_sample(config, device=device), call.CallSampleError)


def _main_combine(config, log):
    """combine mode (.snf / .tsv inputs): on one GPU, or on the ranks of a torchrun launch with --gpus equal to its world size"""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    refusal = None
    if world > 1 and config.gpus == 1:
        refusal = (f"combine mode (.snf / .tsv input) runs on one GPU: run it without torchrun ({world} ranks would each write {config.vcf}), "
                   f"or pass --gpus {world} to run it on the {world} ranks")
    elif world > 1 and config.gpus != world:
        refusal = _mismatch(config, world)
    elif config.combine_consensus:
        refusal = "--combine-consensus is not supported: the reference's SVGroup.call cannot run with it either (sv.py:387)"
    elif config.dev_population_snf is not None:
        refusal = "--dev-population-snf: writing a population SNF is not supported by sniffles_b200; --combine-population reads one"
    if world > 1 and config.gpus > 1:
        return _launch_ranks(world, log, refusal, lambda device: combine_run.combine_snfs(config, device=device), combine_run.CombineError)
    if refusal is not None:
        log.error(f"{refusal} (Fatal error, exiting.)")
        return 1
    try:
        combine_run.combine_snfs(config)
    except combine_run.CombineError as e:
        log.error(f"{e} (Fatal error, exiting.)")
        return 1
    return 0


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    config = SnifflesConfig(*argv)
    config.start_date = datetime.datetime.now().strftime("%Y/%m/%d %H:%M:%S")
    config.command = " ".join(["sniffles"] + argv)
    log = logging.getLogger("sniffles_b200.main")
    exts = {f.split(".")[-1].lower() for f in config.input}
    if len(exts) > 1:
        log.error(f"Please specify either: A single .bam/.cram file - OR - one or more .snf files - OR - a single .tsv file containing a list of "
                  f".snf files and optional sample ids as input. (supplied were: {list(exts)}) (Fatal error, exiting.)")
        return 1
    if exts <= {"snf", "tsv"}:
        return _main_combine(config, log)
    if exts != {"bam"} or len(config.input) != 1:
        log.error(f"Please specify a single .bam file as input: combine mode (.snf / .tsv) and CRAM input are not run by sniffles_b200 "
                  f"(supplied were: {sorted(exts)}) (Fatal error, exiting.)")
        return 1
    config.input = config.input[0]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        return _main_ranks(config, world, log)
    try:
        if config.mode == "genotype_vcf":
            genotype.genotype_vcf(config)
        else:
            call.call_sample(config)
    except (call.CallSampleError, genotype.TargetVcfError) as e:
        log.error(f"{e} (Fatal error, exiting.)")
        return 1
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(name)s (%(process)d): %(message)s", stream=sys.stdout)
    sys.exit(main())
