#!/usr/bin/env python3
"""Write tests/golden/unicode13.json: the Unicode 13.0 classes Go 1.16 (the reference's toolchain) lexes and quotes with.

  letter  unicode.IsLetter   General_Category L
  number  unicode.IsNumber   General_Category N
  print   strconv.IsPrint    General_Category L, M, N, P or S, and U+0020
  space   unicode.IsSpace    \\t \\n \\v \\f \\r, U+0020, U+0085, U+00A0 in Latin-1 (Go's own rule), White_Space above it

A code point belongs to a class if it was assigned in Unicode 13.0 (`Present_In=13.0`, i.e. Age <= 13.0) and its
category qualifies.  The data is perl's `unicore` (Unicode::UCD::prop_invlist), which carries the Age of every code point,
so no network and no download is needed.  Its General_Category is the installed version's (15.0 with perl 5.38): a code
point that 13.0 already had and whose category changed later is classified by the newer data.

Before writing, the tool checks the data against published totals: the assigned graphic and format characters of
Unicode 13.0, 14.0 and 15.0 (143,859 / 144,697 / 149,186), and the sizes of the four classes in 13.0.

Usage: python tools/extract_unicode13.py   (rewrites tests/golden/unicode13.json; tools/gen_unicode_tables.py reads it)
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "unicode13.json")

PROPS = ["Present_In=13.0", "Present_In=14.0", "Present_In=15.0", "White_Space"] + \
        [f"gc={c}" for c in ("L", "M", "N", "P", "S", "Zs", "Zl", "Zp", "Cf")]

# every property's inversion list on one line "<name>\t<cp> <cp> ...", then the provenance
PERL = r"""
use strict; use warnings;
use Unicode::UCD qw(prop_invlist);
for my $p (@ARGV) {
    my @l = prop_invlist($p);
    die "no inversion list for $p\n" unless @l;
    print "$p\t", join(" ", @l), "\n";
}
printf "perl\t%vd\n", $^V;
print "unicore\t", Unicode::UCD::UnicodeVersion(), "\n";
"""

PUBLISHED_TOTALS = {"13.0": 143859, "14.0": 144697, "15.0": 149186}  # assigned graphic + format characters
EXPECTED_13 = {"letter": 131241, "number": 1781, "print": 143680, "space": 25}
GO_LATIN1_SPACE = {0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0}


def invlist_set(inv):
    """inversion list (starts of alternating in/out runs; an odd length runs to the end of the code space) -> set"""
    out = set()
    for k in range(0, len(inv), 2):
        out.update(range(inv[k], inv[k + 1] if k + 1 < len(inv) else 0x110000))
    return out


def ranges(cps):
    out = []
    for cp in sorted(cps):
        if out and out[-1][1] == cp - 1:
            out[-1][1] = cp
        else:
            out.append([cp, cp])
    return out


def main():
    text = subprocess.run(["perl", "-e", PERL, *PROPS], check=True, capture_output=True, text=True).stdout
    sets, prov = {}, {}
    for line in text.splitlines():
        name, _, rest = line.partition("\t")
        if name in PROPS:
            sets[name] = invlist_set([int(x) for x in rest.split()])
        else:
            prov[name] = rest
    gc = {c: sets[f"gc={c}"] for c in ("L", "M", "N", "P", "S", "Zs", "Zl", "Zp", "Cf")}
    graphic_format = set().union(*gc.values())
    for ver, want in PUBLISHED_TOTALS.items():
        got = len(graphic_format & sets[f"Present_In={ver}"])
        if got != want:
            sys.exit(f"Unicode {ver}: {got} assigned graphic and format characters, the published total is {want}")
    in13 = sets["Present_In=13.0"]
    classes = {
        "letter": gc["L"] & in13,
        "number": gc["N"] & in13,
        "print": ((gc["L"] | gc["M"] | gc["N"] | gc["P"] | gc["S"]) & in13) | {0x20},
        "space": GO_LATIN1_SPACE | {cp for cp in sets["White_Space"] & in13 if cp > 0xFF},
    }
    for name, want in EXPECTED_13.items():
        if len(classes[name]) != want:
            sys.exit(f"{name}: {len(classes[name])} code points in Unicode 13.0, expected {want}")
    lines = ["{",
             f' "source": {json.dumps("perl Unicode::UCD prop_invlist: Present_In=13.0 and General_Category / White_Space")},',
             f' "perl": {json.dumps(prov["perl"])},',
             f' "unicore_version": {json.dumps(prov["unicore"])},',
             f' "counts": {json.dumps({k: len(v) for k, v in classes.items()})},']
    names = list(classes)
    for i, name in enumerate(names):
        sep = "," if i + 1 < len(names) else ""
        lines.append(f' "{name}": {json.dumps(ranges(classes[name]), separators=(",", ":"))}{sep}')
    lines.append("}")
    with open(OUT, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("wrote", os.path.relpath(OUT, ROOT), {k: len(v) for k, v in classes.items()})


if __name__ == "__main__":
    main()
