"""`python -m yomitoku_b200 <file-or-dir> -f md -o results`: see cli.py."""
from .cli import main

if __name__ == "__main__":
    main()
