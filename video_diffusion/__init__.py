"""Drop-in alias of the reference's `video_diffusion` import paths (hard-coded in its YAML configs and test_fatezero.py:24-30),
backed by the H100-native implementation in `fatezero_b200`.  Only the hot-path surface of SURVEY.md §8(b) is provided."""


def _extend_with_reference(pkg_path, pkg_file, sub):
    """Modules this alias does not provide (video_diffusion.common, .data, .pipelines.p2p_validation_loop, ... imported by the
    reference's test_fatezero.py:24-30) resolve to the reference checkout when one is importable: every `<root>/video_diffusion[/sub]`
    directory found on sys.path (or under $FATEZERO_REFERENCE_ROOT) is appended to this package's __path__ AFTER the alias directory,
    so the alias modules win and everything else falls through to the reference's own files."""
    import os
    import sys
    here = os.path.dirname(os.path.abspath(pkg_file))
    roots = [os.environ.get("FATEZERO_REFERENCE_ROOT")] + list(sys.path)
    for r in roots:
        if not r:
            continue
        d = os.path.join(os.path.abspath(r), "video_diffusion", sub) if sub else os.path.join(os.path.abspath(r), "video_diffusion")
        if os.path.isdir(d) and os.path.abspath(d) != here and d not in pkg_path:
            pkg_path.append(d)


_extend_with_reference(__path__, __file__, "")
