"""run_utils -- small helpers of the driver.  Same public names as the reference module
(ctc_fast/run_utils.py:10-91: dump_config, load_config, CfgStruct, get_git_revision,
get_hostname, touch_file, TimeString) because runNNet and the reference's run-management tools import them."""
import json
import pathlib
import re
import socket
import subprocess
import time


def dump_config(cfg, fname):
    """cfg.json: sorted keys, 4-space indent, compact separators -- the layout the reference writes."""
    pathlib.Path(fname).write_text(json.dumps(cfg, sort_keys=True, indent=4, separators=(",", ":")))


def load_config(fname):
    return json.loads(pathlib.Path(fname).read_text())


class CfgStruct(object):
    """Attribute view of a config dict."""

    def __init__(self, **entries):
        vars(self).update(entries)


def get_git_revision():
    try:
        out = subprocess.run(["git", "rev-parse", "--short", "HEAD"], capture_output=True, text=True, timeout=10)
        return out.stdout.strip() if out.returncode == 0 else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def get_hostname():
    return socket.gethostname().partition(".")[0]


def touch_file(fname):
    pathlib.Path(fname).touch()


class TimeString(object):
    """Run-directory name: local time down to the second, YYYYMMDDhhmmss."""

    PATTERN = re.compile(r"\d{14}$")

    def __str__(self):
        return time.strftime("%Y%m%d%H%M%S")

    @classmethod
    def match(cls, s):
        return cls.PATTERN.match(s)
