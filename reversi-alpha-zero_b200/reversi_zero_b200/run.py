"""Command line of the reference (run.py + manager.py):

    python -m reversi_zero_b200.run {self,opt,eval,nboard,league,openings,book} [-c config.yml] [--new] [--total-step N]

``self`` plays games, ``opt`` trains, ``eval`` promotes, ``nboard`` speaks the NBoard protocol on stdin / stdout,
``league`` rates saved models against each other (settings in the YAML ``league:`` section), ``openings`` writes a suite
of balanced openings for ``eval`` and ``league`` (settings in the YAML ``openings:`` section), ``book`` builds an opening
book for NBoard and for suites (settings in the YAML ``book:`` section).
Files go under the project directory: ``$PROJECT_DIR``, else the current directory.  Every command logs to
``logs/main.log``; all but ``nboard`` also log to stderr.
"""
import argparse
from logging import StreamHandler, basicConfig, DEBUG, getLogger, Formatter

from .config import create_config, load_yaml

logger = getLogger(__name__)

CMD_LIST = ['self', 'opt', 'eval', 'nboard', 'league', 'openings', 'book']


def create_parser():
    parser = argparse.ArgumentParser(prog="python -m reversi_zero_b200.run")
    parser.add_argument("cmd", help="what to do", choices=CMD_LIST)
    parser.add_argument("-c", help="specify config yaml", dest="config_file")
    parser.add_argument("--new", help="run from new best model", action="store_true")
    parser.add_argument("--type", help="deprecated. Please use -c instead")
    parser.add_argument("--total-step", help="set TrainerConfig.start_total_steps", type=int)
    return parser


def setup_logger(log_filename):
    """lib/logger.py: DEBUG and up to the log file, and a copy to stderr"""
    format_str = '%(asctime)s@%(name)s %(levelname)s # %(message)s'
    basicConfig(filename=log_filename, level=DEBUG, format=format_str)
    stream_handler = StreamHandler()
    stream_handler.setFormatter(Formatter(format_str))
    getLogger().addHandler(stream_handler)


def setup(config, args):
    """manager.py:26-31"""
    config.opts.new = args.new
    if args.total_step is not None:
        tr = getattr(config, "trainer", None)
        if tr is None:
            config.trainer = tr = {}
        if isinstance(tr, dict):
            tr["start_total_steps"] = args.total_step
        else:
            tr.start_total_steps = args.total_step
    config.resource.create_directories()
    setup_logger(config.resource.main_log_path)


def load_config(args):
    return load_yaml(args.config_file) if args.config_file else create_config()


def start(argv=None):
    args = create_parser().parse_args(argv)
    if args.type:
        print("I'm very sorry. --type option was deprecated. Please use -c option instead!")
        return 1
    config = load_config(args)
    setup(config, args)

    if args.cmd != "nboard":
        logger.info(f"config type: {config.type}")

    if args.cmd == "self":
        from .worker import self_play
        return self_play.start(config)
    elif args.cmd == 'opt':
        from .worker import optimize
        return optimize.start(config)
    elif args.cmd == 'eval':
        from .worker import evaluate
        return evaluate.start(config)
    elif args.cmd == 'nboard':
        from .play_game import nboard
        return nboard.start(config)
    elif args.cmd == 'league':
        from .worker import league
        return league.start(config)
    elif args.cmd == 'openings':
        from .lib import openings
        return openings.start(config)
    elif args.cmd == 'book':
        from .lib import book
        return book.start(config)


if __name__ == "__main__":
    start()
