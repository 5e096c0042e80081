import sys

from .cli import exit_status, main

sys.exit(exit_status(main()))
