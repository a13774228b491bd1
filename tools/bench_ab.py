"""Alternate `bench.py` between two built trees (A B A B ...) in one session and print every JSON line, so that a difference can be
set against the run-to-run spread.    python tools/bench_ab.py TREE_A TREE_B [runs] [-- bench.py arguments]"""
import subprocess
import sys


def main():
    args = sys.argv[1:]
    extra = ['--gpus', '1', '--steps', '10', '--warmup', '3', '--no-cpu-baseline']
    if '--' in args:
        extra = args[args.index('--') + 1:]
        args = args[:args.index('--')]
    trees = args[:2]
    runs = int(args[2]) if len(args) > 2 else 3
    for i in range(runs):
        for t in trees:
            out = subprocess.run([sys.executable, 'bench.py'] + extra, cwd=t, capture_output=True, text=True)
            lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
            if out.returncode or not lines:
                sys.exit('bench.py failed in %s:\n%s' % (t, out.stderr[-2000:]))
            print('%s run %d: %s' % (t, i, lines[-1]), flush=True)


if __name__ == '__main__':
    main()
