"""Fall-through to the reference tree for everything OUTSIDE the accelerated hot path.

The drop-in package shadows only the modules SURVEY.md section 8(b) lists; `offpolicy.runner`, `offpolicy.envs`,
`offpolicy.config`, `offpolicy.scripts` and the remaining
`offpolicy.utils.*` helpers keep coming, byte-identical, from the reference checkout when one is present
(OFFPOLICY_REFERENCE_ROOT, default /root/reference).  Without a checkout the hot-path modules still work standalone.
"""
import os


def reference_root():
    root = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
    pkg = os.path.join(root, "offpolicy")
    return pkg if os.path.isdir(pkg) else None


def extend(path_list, *sub):
    root = reference_root()
    if root is None:
        return
    d = os.path.join(root, *sub)
    if os.path.isdir(d) and d not in path_list:
        path_list.append(d)
