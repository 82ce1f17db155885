"""evals.scaffold.main: dispatch to evals.<name>.eval.main (reference: evals/scaffold.py:16-24)."""
import importlib
import logging
import sys

logging.basicConfig(stream=sys.stdout, level=logging.INFO)
logger = logging.getLogger()


def main(eval_name, args_eval, resume_preempt=False):
    logger.info(f'Running evaluation: {eval_name}')
    return importlib.import_module(f'evals.{eval_name}.eval').main(args_eval=args_eval, resume_preempt=resume_preempt)
