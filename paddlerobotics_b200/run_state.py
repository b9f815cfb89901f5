"""The --save_state / --resume contract of the training commands (train, pretrain, bctrain, dynamic_train; DESIGN §8g).

    write_atomic(path, obj)     the state file, replaced through a temporary file, fsync and rename
    load_state(p, path, cmd)    the saved state of a --resume, refused (p.error) when another command wrote it
    resume_args(...)            the saved run's arguments with the command's changeable flags from this command line

Every file records the command that wrote it under "command"; a file without that key is train's (written before the key existed).
All refusals are argument errors raised before any device work."""
import argparse
import os

import torch


def write_atomic(path, obj):
    """torch.save(obj) to path through a temporary file that is flushed, fsynced and renamed over it: a crash mid-write leaves the
    previous file intact."""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        torch.save(obj, f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)
    fd = os.open(os.path.dirname(os.path.abspath(path)), os.O_RDONLY)
    try:
        os.fsync(fd)                                                        # the rename itself
    finally:
        os.close(fd)


def command_of(state):
    """The command that wrote a state file: its "command" key, or "train" for a file without one."""
    return state.get("command", "train")


def load_state(p, path, command):
    """The state file of `--resume path` on the CPU; an argument error when `command` did not write it."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if command_of(state) != command:
        p.error("--resume %s: a state file of %s, not of %s" % (path, command_of(state), command))
    return state


def resume_args(p, make_parser, argv, saved, free, conflicts, restores):
    """The arguments of a --resume run: the saved run's, with the `free` flags of this command line.  Any other flag given on the command
    line with a value other than the saved one is an argument error (p.error) naming the flags, as is every (label, dest) of `conflicts`
    that the command line sets (to anything but "", "None" or 0): the flags that set what the state restores (`restores`, for the
    message).  make_parser() builds a fresh parser of the command, whose defaults are dropped to see which flags the command line gave."""
    q = make_parser()
    for a in q._actions:
        a.default = argparse.SUPPRESS
    given = vars(q.parse_args(argv))
    bad = [label for label, dest in conflicts if given.get(dest, "") not in ("", "None", 0)]
    if bad:
        p.error("--resume restores %s: it cannot be combined with %s" % (restores, ", ".join(bad)))
    differ = sorted(k for k, v in given.items() if k not in free and v != saved.get(k))
    if differ:
        p.error("--resume %s: these arguments differ from the saved run's: %s" % (given["resume"], ", ".join("--" + k for k in differ)))
    args = argparse.Namespace(**saved)
    for k in free:
        if k in given:
            setattr(args, k, given[k])
    return args
