"""`python -m bonito_b200 <subcommand>`: argparse sub-command dispatch as in `bonito/__init__.py:14-32`."""
from argparse import ArgumentParser, ArgumentDefaultsHelpFormatter

from bonito_b200 import __version__
from bonito_b200.cli import basecaller, duplex, evaluate, train

modules = ["basecaller", "duplex", "evaluate", "train"]


def main():
    parser = ArgumentParser("bonito_b200", formatter_class=ArgumentDefaultsHelpFormatter)
    parser.add_argument("-v", "--version", action="version", version="%(prog)s {}".format(__version__))
    subparsers = parser.add_subparsers(title="subcommands", description="valid commands", help="additional help",
                                       dest="command")
    subparsers.required = True
    for name, mod in (("basecaller", basecaller), ("duplex", duplex), ("evaluate", evaluate), ("train", train)):
        p = subparsers.add_parser(name, parents=[mod.argparser()])
        p.set_defaults(func=mod.main)
    args = parser.parse_args()
    args.func(args)


if __name__ == "__main__":
    main()
