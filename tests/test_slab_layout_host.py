"""Where ``coda.datasets.Dataset`` (main.py's loader) loads a task file, on the CPU: every combination of the
``CODA_B200_*`` settings, the visible GPUs, their free memory and the file's format, against a literal table of the
load each one gets."""
import re

import pytest
import torch

H, N, C = 4, 50, 10
BIG = 1 << 50

HOST_SLAB = (None, "", "0", "1")
SHARD_LOAD = (None, "", "0", "1")
# free bytes of each visible GPU: everything fits, only the target GPU (cuda:0) is too small, every GPU is too small,
# or torch.cuda.mem_get_info fails
FREE = {"fits": lambda n: [BIG] * n, "target": lambda n: [0] + [BIG] * (n - 1), "sum": lambda n: [0] * n,
        "error": None}
DEFAULTS = {"keep_dtype": False, "shards": None, "gpus": None, "compact_k": None, "host": False}

# (file, visible GPUs, free memory, CODA_B200_GPUS, CODA_B200_COMPACT_K) -> the load of each CODA_B200_HOST_SLAB value
# (unset | "" | "0" | "1"), each a row over CODA_B200_SHARD_LOAD (unset, "", "0", "1").  A load is its arguments that
# differ from their defaults: k keep_dtype=True, h host=True, c<K> compact_k=K, s<n> shards=n, "-" none of them; or
# what the shim raises: "!" a RuntimeError, else the exception's name.
TABLE = {
    ('dense32', 1, 'fits', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('dense32', 1, 'fits', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense32', 1, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('dense32', 1, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 1, 'target', None, None): 'h h h h | h h h h | - - - s1 | h h h h',
    ('dense32', 1, 'target', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense32', 1, 'target', '3', None): 'h h h h | h h h h | - - - s3 | h h h h',
    ('dense32', 1, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 1, 'sum', None, None): 'h h h h | h h h h | - - - s1 | h h h h',
    ('dense32', 1, 'sum', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense32', 1, 'sum', '3', None): 'h h h h | h h h h | - - - s3 | h h h h',
    ('dense32', 1, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 1, 'error', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('dense32', 1, 'error', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense32', 1, 'error', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('dense32', 1, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 2, 'fits', None, None): '- - - s2 | - - - s2 | - - - s2 | h h h h',
    ('dense32', 2, 'fits', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('dense32', 2, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('dense32', 2, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 2, 'target', None, None): 's2 s2 s2 s2 | s2 s2 s2 s2 | s2 s2 s2 s2 | h h h h',
    ('dense32', 2, 'target', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('dense32', 2, 'target', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | h h h h',
    ('dense32', 2, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense32', 2, 'sum', None, None): 'hs2 hs2 s2 s2 | hs2 hs2 s2 s2 | s2 s2 s2 s2 | h h h h',
    ('dense32', 2, 'sum', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('dense32', 2, 'sum', '3', None): 'hs3 hs3 s3 s3 | hs3 hs3 s3 s3 | s3 s3 s3 s3 | h h h h',
    ('dense32', 2, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense32', 2, 'error', None, None): '! ! ! s2 | ! ! ! s2 | ! ! ! s2 | h h h h',
    ('dense32', 2, 'error', None, '4'): '! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2',
    ('dense32', 2, 'error', '3', None): '! ! ! s3 | ! ! ! s3 | ! ! ! s3 | h h h h',
    ('dense32', 2, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
    ('dense32', 4, 'fits', None, None): '- - - s4 | - - - s4 | - - - s4 | h h h h',
    ('dense32', 4, 'fits', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('dense32', 4, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('dense32', 4, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense32', 4, 'target', None, None): 's4 s4 s4 s4 | s4 s4 s4 s4 | s4 s4 s4 s4 | h h h h',
    ('dense32', 4, 'target', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('dense32', 4, 'target', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | h h h h',
    ('dense32', 4, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense32', 4, 'sum', None, None): 'hs4 hs4 s4 s4 | hs4 hs4 s4 s4 | s4 s4 s4 s4 | h h h h',
    ('dense32', 4, 'sum', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('dense32', 4, 'sum', '3', None): 'hs3 hs3 s3 s3 | hs3 hs3 s3 s3 | s3 s3 s3 s3 | h h h h',
    ('dense32', 4, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense32', 4, 'error', None, None): '! ! ! s4 | ! ! ! s4 | ! ! ! s4 | h h h h',
    ('dense32', 4, 'error', None, '4'): '! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4',
    ('dense32', 4, 'error', '3', None): '! ! ! s3 | ! ! ! s3 | ! ! ! s3 | h h h h',
    ('dense32', 4, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
    ('dense16_keep', 1, 'fits', None, None): 'k k k ks1 | k k k ks1 | k k k ks1 | kh kh kh kh',
    ('dense16_keep', 1, 'fits', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense16_keep', 1, 'fits', '3', None): 'k k k ks3 | k k k ks3 | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 1, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 1, 'target', None, None): 'kh kh kh kh | kh kh kh kh | k k k ks1 | kh kh kh kh',
    ('dense16_keep', 1, 'target', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense16_keep', 1, 'target', '3', None): 'kh kh kh kh | kh kh kh kh | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 1, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 1, 'sum', None, None): 'kh kh kh kh | kh kh kh kh | k k k ks1 | kh kh kh kh',
    ('dense16_keep', 1, 'sum', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense16_keep', 1, 'sum', '3', None): 'kh kh kh kh | kh kh kh kh | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 1, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 1, 'error', None, None): 'k k k ks1 | k k k ks1 | k k k ks1 | kh kh kh kh',
    ('dense16_keep', 1, 'error', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('dense16_keep', 1, 'error', '3', None): 'k k k ks3 | k k k ks3 | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 1, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 2, 'fits', None, None): 'k k k ks2 | k k k ks2 | k k k ks2 | kh kh kh kh',
    ('dense16_keep', 2, 'fits', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('dense16_keep', 2, 'fits', '3', None): 'k k k ks3 | k k k ks3 | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 2, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 2, 'target', None, None): 'ks2 ks2 ks2 ks2 | ks2 ks2 ks2 ks2 | ks2 ks2 ks2 ks2 | kh kh kh kh',
    ('dense16_keep', 2, 'target', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('dense16_keep', 2, 'target', '3', None): 'ks3 ks3 ks3 ks3 | ks3 ks3 ks3 ks3 | ks3 ks3 ks3 ks3 | kh kh kh kh',
    ('dense16_keep', 2, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense16_keep', 2, 'sum', None, None): 'khs2 khs2 ks2 ks2 | khs2 khs2 ks2 ks2 | ks2 ks2 ks2 ks2 | kh kh kh kh',
    ('dense16_keep', 2, 'sum', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('dense16_keep', 2, 'sum', '3', None): 'khs3 khs3 ks3 ks3 | khs3 khs3 ks3 ks3 | ks3 ks3 ks3 ks3 | kh kh kh kh',
    ('dense16_keep', 2, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense16_keep', 2, 'error', None, None): '! ! ! ks2 | ! ! ! ks2 | ! ! ! ks2 | kh kh kh kh',
    ('dense16_keep', 2, 'error', None, '4'): '! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2',
    ('dense16_keep', 2, 'error', '3', None): '! ! ! ks3 | ! ! ! ks3 | ! ! ! ks3 | kh kh kh kh',
    ('dense16_keep', 2, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
    ('dense16_keep', 4, 'fits', None, None): 'k k k ks4 | k k k ks4 | k k k ks4 | kh kh kh kh',
    ('dense16_keep', 4, 'fits', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('dense16_keep', 4, 'fits', '3', None): 'k k k ks3 | k k k ks3 | k k k ks3 | kh kh kh kh',
    ('dense16_keep', 4, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('dense16_keep', 4, 'target', None, None): 'ks4 ks4 ks4 ks4 | ks4 ks4 ks4 ks4 | ks4 ks4 ks4 ks4 | kh kh kh kh',
    ('dense16_keep', 4, 'target', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('dense16_keep', 4, 'target', '3', None): 'ks3 ks3 ks3 ks3 | ks3 ks3 ks3 ks3 | ks3 ks3 ks3 ks3 | kh kh kh kh',
    ('dense16_keep', 4, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense16_keep', 4, 'sum', None, None): 'khs4 khs4 ks4 ks4 | khs4 khs4 ks4 ks4 | ks4 ks4 ks4 ks4 | kh kh kh kh',
    ('dense16_keep', 4, 'sum', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('dense16_keep', 4, 'sum', '3', None): 'khs3 khs3 ks3 ks3 | khs3 khs3 ks3 ks3 | ks3 ks3 ks3 ks3 | kh kh kh kh',
    ('dense16_keep', 4, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('dense16_keep', 4, 'error', None, None): '! ! ! ks4 | ! ! ! ks4 | ! ! ! ks4 | kh kh kh kh',
    ('dense16_keep', 4, 'error', None, '4'): '! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4',
    ('dense16_keep', 4, 'error', '3', None): '! ! ! ks3 | ! ! ! ks3 | ! ! ! ks3 | kh kh kh kh',
    ('dense16_keep', 4, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
    ('legacy', 1, 'fits', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('legacy', 1, 'fits', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('legacy', 1, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 1, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 1, 'target', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('legacy', 1, 'target', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('legacy', 1, 'target', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 1, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 1, 'sum', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('legacy', 1, 'sum', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('legacy', 1, 'sum', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 1, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 1, 'error', None, None): '- - - s1 | - - - s1 | - - - s1 | h h h h',
    ('legacy', 1, 'error', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('legacy', 1, 'error', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 1, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 2, 'fits', None, None): '- - - s2 | - - - s2 | - - - s2 | h h h h',
    ('legacy', 2, 'fits', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('legacy', 2, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 2, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 2, 'target', None, None): '- - - s2 | - - - s2 | - - - s2 | h h h h',
    ('legacy', 2, 'target', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('legacy', 2, 'target', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 2, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 2, 'sum', None, None): '- - - s2 | - - - s2 | - - - s2 | h h h h',
    ('legacy', 2, 'sum', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('legacy', 2, 'sum', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 2, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 2, 'error', None, None): '- - - s2 | - - - s2 | - - - s2 | h h h h',
    ('legacy', 2, 'error', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('legacy', 2, 'error', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 2, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 4, 'fits', None, None): '- - - s4 | - - - s4 | - - - s4 | h h h h',
    ('legacy', 4, 'fits', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('legacy', 4, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 4, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 4, 'target', None, None): '- - - s4 | - - - s4 | - - - s4 | h h h h',
    ('legacy', 4, 'target', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('legacy', 4, 'target', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 4, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 4, 'sum', None, None): '- - - s4 | - - - s4 | - - - s4 | h h h h',
    ('legacy', 4, 'sum', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('legacy', 4, 'sum', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 4, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('legacy', 4, 'error', None, None): '- - - s4 | - - - s4 | - - - s4 | h h h h',
    ('legacy', 4, 'error', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('legacy', 4, 'error', '3', None): '- - - s3 | - - - s3 | - - - s3 | h h h h',
    ('legacy', 4, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 1, 'fits', None, None): '- - - s1 | - - - s1 | - - - s1 | - - - s1',
    ('compact', 1, 'fits', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('compact', 1, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 1, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 1, 'target', None, None): '- - - s1 | - - - s1 | - - - s1 | - - - s1',
    ('compact', 1, 'target', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('compact', 1, 'target', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 1, 'target', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 1, 'sum', None, None): '- - - s1 | - - - s1 | - - - s1 | - - - s1',
    ('compact', 1, 'sum', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('compact', 1, 'sum', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 1, 'sum', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 1, 'error', None, None): '- - - s1 | - - - s1 | - - - s1 | - - - s1',
    ('compact', 1, 'error', None, '4'): 'c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1 | c4 c4 c4 c4s1',
    ('compact', 1, 'error', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 1, 'error', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 2, 'fits', None, None): '- - - s2 | - - - s2 | - - - s2 | - - - s2',
    ('compact', 2, 'fits', None, '4'): 'c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2 | c4 c4 c4 c4s2',
    ('compact', 2, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 2, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 2, 'target', None, None): 's2 s2 s2 s2 | s2 s2 s2 s2 | s2 s2 s2 s2 | s2 s2 s2 s2',
    ('compact', 2, 'target', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('compact', 2, 'target', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3',
    ('compact', 2, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('compact', 2, 'sum', None, None): 's2 s2 s2 s2 | s2 s2 s2 s2 | s2 s2 s2 s2 | s2 s2 s2 s2',
    ('compact', 2, 'sum', None, '4'):
        'c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2 | c4s2 c4s2 c4s2 c4s2',
    ('compact', 2, 'sum', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3',
    ('compact', 2, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('compact', 2, 'error', None, None): '! ! ! s2 | ! ! ! s2 | ! ! ! s2 | ! ! ! s2',
    ('compact', 2, 'error', None, '4'): '! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2 | ! ! ! c4s2',
    ('compact', 2, 'error', '3', None): '! ! ! s3 | ! ! ! s3 | ! ! ! s3 | ! ! ! s3',
    ('compact', 2, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
    ('compact', 4, 'fits', None, None): '- - - s4 | - - - s4 | - - - s4 | - - - s4',
    ('compact', 4, 'fits', None, '4'): 'c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4 | c4 c4 c4 c4s4',
    ('compact', 4, 'fits', '3', None): '- - - s3 | - - - s3 | - - - s3 | - - - s3',
    ('compact', 4, 'fits', '3', '4'): 'c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3 | c4 c4 c4 c4s3',
    ('compact', 4, 'target', None, None): 's4 s4 s4 s4 | s4 s4 s4 s4 | s4 s4 s4 s4 | s4 s4 s4 s4',
    ('compact', 4, 'target', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('compact', 4, 'target', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3',
    ('compact', 4, 'target', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('compact', 4, 'sum', None, None): 's4 s4 s4 s4 | s4 s4 s4 s4 | s4 s4 s4 s4 | s4 s4 s4 s4',
    ('compact', 4, 'sum', None, '4'):
        'c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4 | c4s4 c4s4 c4s4 c4s4',
    ('compact', 4, 'sum', '3', None): 's3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3 | s3 s3 s3 s3',
    ('compact', 4, 'sum', '3', '4'):
        'c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3 | c4s3 c4s3 c4s3 c4s3',
    ('compact', 4, 'error', None, None): '! ! ! s4 | ! ! ! s4 | ! ! ! s4 | ! ! ! s4',
    ('compact', 4, 'error', None, '4'): '! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4 | ! ! ! c4s4',
    ('compact', 4, 'error', '3', None): '! ! ! s3 | ! ! ! s3 | ! ! ! s3 | ! ! ! s3',
    ('compact', 4, 'error', '3', '4'): '! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3 | ! ! ! c4s3',
}


def _files(tmp_path):
    from coda_b200 import CompactSlab
    torch.manual_seed(0)
    t = torch.rand(H, N, C)
    paths = {k: str(tmp_path / f"{k}.pt") for k in ("dense32", "dense16_keep", "legacy", "compact")}
    torch.save(t, paths["dense32"])
    torch.save(t.half(), paths["dense16_keep"])
    torch.save(t, paths["legacy"], _use_new_zipfile_serialization=False)
    top = t.topk(3, dim=2)
    CompactSlab(top.indices.to(torch.int16), top.values, C).save(paths["compact"])
    return paths


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return _files(tmp_path_factory.mktemp("slab_layout"))


def _load(monkeypatch, path, env, ngpus, free):
    """The effective arguments the shim passes to ``coda_b200.datasets.Dataset``, as a token string."""
    import coda_b200.datasets as ds
    from coda.datasets import Dataset
    for k in ("CODA_B200_HOST_SLAB", "CODA_B200_SHARD_LOAD", "CODA_B200_GPUS", "CODA_B200_COMPACT_K",
              "CODA_B200_KEEP_DTYPE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        if v is not None:
            monkeypatch.setenv(k, v)
    per_gpu = FREE[free]

    def mem_get_info(index):
        if per_gpu is None:
            raise RuntimeError("mem_get_info failed")
        return per_gpu(ngpus)[index], BIG

    monkeypatch.setattr(torch.cuda, "mem_get_info", mem_get_info)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: ngpus)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    calls = []
    monkeypatch.setattr(ds.Dataset, "__init__", lambda self, *a, **kw: calls.append((a, kw)))
    try:
        Dataset(path, "cuda:0")
    except Exception as e:                                          # noqa: BLE001 -- the outcome is the exception
        return "!" if type(e) is RuntimeError else type(e).__name__
    (args, kw), = calls
    assert args == (path, "cuda:0")
    kw = {k: v for k, v in kw.items() if v != DEFAULTS[k]}
    out = ("k" if kw.pop("keep_dtype", False) else "") + ("h" if kw.pop("host", False) else "")
    if "compact_k" in kw:
        out += f"c{kw.pop('compact_k')}"
    if "shards" in kw:
        out += f"s{kw.pop('shards')}"
    assert not kw, kw
    return out or "-"


def _row(monkeypatch, paths, file, ngpus, free, gpus, k):
    groups = []
    for hs in HOST_SLAB:
        loads = []
        for sl in SHARD_LOAD:
            env = {"CODA_B200_HOST_SLAB": hs, "CODA_B200_SHARD_LOAD": sl, "CODA_B200_GPUS": gpus,
                   "CODA_B200_COMPACT_K": k, "CODA_B200_KEEP_DTYPE": "1" if file == "dense16_keep" else None}
            loads.append(_load(monkeypatch, paths[file], env, ngpus, free))
        groups.append(" ".join(loads))
    return " | ".join(groups)


@pytest.mark.parametrize("key", list(TABLE), ids=lambda key: "-".join(str(x) for x in key))
def test_shim_load_route(files, monkeypatch, key):
    assert _row(monkeypatch, files, *key) == TABLE[key]


def test_table_covers_every_combination():
    keys = [(f, g, fr, gp, k) for f in ("dense32", "dense16_keep", "legacy", "compact") for g in (1, 2, 4)
            for fr in FREE for gp in (None, "3") for k in (None, "4")]
    assert sorted(TABLE, key=str) == sorted(keys, key=str)
    assert all(re.fullmatch(r"(\S+ ){3}\S+( \| (\S+ ){3}\S+){3}", v) for v in TABLE.values())
