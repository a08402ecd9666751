"""Every measurement file the documents cite exists under profiles/ (evidence links must not rot)."""
import glob
import os
import re

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOCS = ["README.md", "BASELINE.md"] + sorted(
    os.path.relpath(p, REPO) for p in glob.glob(os.path.join(REPO, "docs", "source", "**", "*.md"), recursive=True))


def _expand(text):
    """`a_{x,y}.json` → a_x.json, a_y.json (the shorthand the tables use)."""
    out = text
    for m in re.finditer(r"([\w\-./]*)\{([^{}`]*)\}([\w\-.]*)", text):
        out += " " + " ".join(m.group(1) + alt.strip() + m.group(3) for alt in m.group(2).split(","))
    return out


def test_cited_profile_files_exist():
    missing = []
    for doc in DOCS:
        path = os.path.join(REPO, doc)
        assert os.path.exists(path), doc
        text = _expand(open(path).read())
        names = set(re.findall(r"\b(r2?_?\d+_[\w\-.]+\.(?:json|md|txt|log))\b", text))
        names |= set(re.findall(r"\bprofiles/([\w\-./*]+)", text))
        for name in names:
            hits = glob.glob(os.path.join(REPO, "profiles", name)) + glob.glob(os.path.join(REPO, "profiles", "sanitizer", name))
            if not hits:
                missing.append((doc, name))
    assert not missing, missing
