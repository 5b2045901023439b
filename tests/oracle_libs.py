"""Module-scoped fixtures on the CPU checkers of oracle/ (oracle.load): `refc` (libsvtav1_ref.so) and one per checker
library.  A test module imports the ones it uses, under the fixture name it wants (pytest names a fixture after the
module attribute: `from oracle_libs import dlf as dlfc`); an imported `refc` overrides conftest.py's for that module.

A library that is not built fails every test of the module that requests it when one of the selected tests that do is
marked gpu -- a parity test must never pass by skipping -- and skips them otherwise: the CPU pins may run on a clone
without the reference sources."""
import oracle
import pytest


def library(name):
    """a module-scoped fixture on oracle.load(name)"""
    @pytest.fixture(scope="module")
    def fixture(request):
        lib = oracle.load(name)
        if lib is None:
            users = [it for it in request.session.items
                     if request.node in it.listchain() and request.fixturename in it.fixturenames]
            msg = "oracle/_ref/%s is missing" % oracle.LIBS[name]
            if any(it.get_closest_marker("gpu") is not None for it in users):
                pytest.fail("%s: %s" % (msg, oracle.BUILD_HINT))
            pytest.skip("%s (the reference sources are not available)" % msg)
        return lib
    return fixture


refc = library("ref")
dlf = library("dlf")
dlf_search = library("dlf_search")
pa_stats = library("pa_stats")
enc = library("enc")
