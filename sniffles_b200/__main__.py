"""`python -m sniffles_b200 ARGS`: the reference's command line (sniffles:64-148) for the two run modes that read one BAM -- calling a
sample (`-i sample.bam -v out.vcf [--snf out.snf]`, call.call_sample) and force calling (`--genotype-vcf`, genotype.genotype_vcf).
Combine mode (.snf / .tsv input) and CRAM input are not run from here."""
import datetime
import logging
import sys

from . import call, genotype
from .config import SnifflesConfig


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    config = SnifflesConfig(*argv)
    config.start_date = datetime.datetime.now().strftime("%Y/%m/%d %H:%M:%S")
    config.command = " ".join(["sniffles"] + argv)
    log = logging.getLogger("sniffles_b200.main")
    exts = {f.split(".")[-1].lower() for f in config.input}
    if exts != {"bam"} or len(config.input) != 1:
        log.error(f"Please specify a single .bam file as input: combine mode (.snf / .tsv) and CRAM input are not run by sniffles_b200 "
                  f"(supplied were: {sorted(exts)}) (Fatal error, exiting.)")
        return 1
    config.input = config.input[0]
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
