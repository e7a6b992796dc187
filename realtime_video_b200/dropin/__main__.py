"""``python -m realtime_video_b200.dropin <script.py | -m module> [args...]`` — run an unmodified reference entry
point (sample.py, ``-m uvicorn release_server:app`` ...) with this package's classes behind the reference's import names."""
import runpy
import sys

from . import install


def main(argv):
    if not argv:
        print(__doc__)
        return 2
    install()
    if argv[0] == "-m":
        if len(argv) < 2:
            print(__doc__)
            return 2
        sys.argv = argv[1:]
        if "" not in sys.path:
            sys.path.insert(0, "")                  # what ``python -m`` does
        runpy.run_module(argv[1], run_name="__main__", alter_sys=True)
    else:
        import os
        sys.argv = argv
        sys.path.insert(0, os.path.dirname(os.path.abspath(argv[0])))   # what ``python script.py`` does
        runpy.run_path(argv[0], run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
