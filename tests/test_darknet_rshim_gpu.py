"""The R shim of image.darknet (image_b200/rshim/darknet_r_api.c) against the package's own R glue (src/__R_API_*.c,
built unmodified into oracle/_ref/libref_darknet_rapi.so).  Both are compiled against the R stubs of oracle/stubs/ into
one small program each, which calls the .Call entry points darknet_detect and darknet_predict with stub SEXPs.  The
printed lines (draw_detections' labels and percentages, the box count), predictions.png and the returned labels and
scores must be identical; only the timing in "Predicted in ... seconds" may differ."""
import os
import re
import subprocess

import pytest

from oracle import ref_darknet as rd
from darknet_cases import random_weights, shrink_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
INC = os.path.join(REF, "darknet", "include")
RAPI = os.path.join(REF, "libref_darknet_rapi.so")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (rd.have_ref() and os.path.exists(RAPI) and os.path.isdir(INC)),
                                                  reason="reference build of image.darknet and its R glue absent")]

HARNESS = r"""
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <Rinternals.h>
SEXP darknet_detect(SEXP, SEXP, SEXP, SEXP, SEXP, SEXP, SEXP);
SEXP darknet_predict(SEXP, SEXP, SEXP, SEXP, SEXP, SEXP, SEXP);
static SEXP str(const char *s) { SEXP v = allocVector(STRSXP, 1); SET_STRING_ELT(v, 0, mkChar(s)); return v; }
static SEXP num(double d) { SEXP v = allocVector(REALSXP, 1); REAL(v)[0] = d; return v; }
static SEXP integer(int i) { SEXP v = allocVector(INTSXP, 1); INTEGER(v)[0] = i; return v; }
static SEXP lines(const char *file) {
  static char buf[1 << 16][64];
  int n = 0;
  FILE *f = fopen(file, "r");
  while (n < (1 << 16) && fgets(buf[n], 64, f)) { buf[n][strcspn(buf[n], "\n")] = 0; n++; }
  fclose(f);
  SEXP v = allocVector(STRSXP, n);
  for (int i = 0; i < n; i++) SET_STRING_ELT(v, i, mkChar(buf[i]));
  return v;
}
/* detect cfg weights image labels root thresh hier | classify cfg weights image labels top resize */
int main(int argc, char **argv) {
  if (!strcmp(argv[1], "detect")) {
    SEXP r = darknet_detect(str(argv[2]), str(argv[3]), str(argv[4]), num(atof(argv[7])), num(atof(argv[8])), lines(argv[5]),
                            str(argv[6]));
    printf("returned %s\n", CHAR(STRING_ELT(r, 0)));
  } else {
    SEXP r = darknet_predict(str("not_needed_any_more.data"), str(argv[2]), str(argv[3]), str(argv[4]), integer(atoi(argv[6])),
                             lines(argv[5]), integer(atoi(argv[7])));
    SEXP sc = VECTOR_ELT(r, 0), lb = VECTOR_ELT(r, 1);
    for (int i = 0; i < LENGTH(sc); i++) printf("%s %a\n", CHAR(STRING_ELT(lb, i)), REAL(sc)[i]);
  }
  fflush(stdout);
  return 0;
}
"""


@pytest.fixture(scope="module")
def programs(tmp_path_factory):
    d = tmp_path_factory.mktemp("dnshim")
    src = d / "harness.c"
    src.write_text(HARNESS)
    common = ["-O1", "-I" + os.path.join(ROOT, "oracle", "stubs"), "-I" + INC, "-I" + os.path.join(ROOT, "include"), str(src)]
    rpath = "-Wl,-rpath," + REF + ":" + os.path.join(ROOT, "image_b200")
    shim, ref = str(d / "shim"), str(d / "ref")
    subprocess.check_call(["gcc"] + common + [os.path.join(ROOT, "image_b200", "rshim", "darknet_r_api.c"),
                                              "-L" + REF, "-lref_darknet", "-L" + os.path.join(ROOT, "image_b200"), "-lb200feat",
                                              rpath, "-lm", "-o", shim])
    subprocess.check_call(["gcc"] + common + ["-L" + REF, "-lref_darknet_rapi", "-lref_darknet", rpath, "-lm", "-o", ref])
    return shim, ref


def run(prog, args, cwd):
    os.makedirs(cwd, exist_ok=True)
    out = subprocess.run([prog] + [str(a) for a in args], cwd=cwd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return re.sub(r"Predicted in [0-9.]+ seconds", "Predicted in - seconds", out.stdout)


def same(programs, args, tmp_path, png=False):
    shim, ref = programs
    a, b = run(shim, args, str(tmp_path / "shim")), run(ref, args, str(tmp_path / "ref"))
    assert a == b
    if png:
        with open(tmp_path / "shim" / "predictions.png", "rb") as f1, open(tmp_path / "ref" / "predictions.png", "rb") as f2:
            assert f1.read() == f2.read()
    return a


@pytest.mark.parametrize("name", ["dog.jpg", "horses.jpg", "person.jpg"])
def test_detect_shim_prints_and_draws_the_reference_detections(programs, tmp_path, name):
    out = same(programs, ["detect", rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"), rd.path(name),
                          rd.path("voc.names"), os.path.join(REF, "darknet"), 0.3, 0.5], tmp_path, png=True)
    if name == "dog.jpg":
        assert "dog: 79%" in out and "car: 76%" in out and "Boxes: 845 of which 2 above the threshold." in out


@pytest.mark.parametrize("resize", [1, 0])
@pytest.mark.parametrize("name", ["eagle.jpg", "giraffe.jpg"])
def test_classify_shim_returns_the_reference_labels_and_scores(programs, tmp_path, name, resize):
    out = same(programs, ["classify", rd.path("tiny.cfg"), rd.path("tiny.weights"), rd.path(name),
                          rd.path("imagenet.shortnames.list"), 5, resize], tmp_path)
    assert len(out.splitlines()) == 5


def test_unsupported_cfg_keeps_the_reference_forward_pass(programs, tmp_path):
    """yolo-voc has route and reorg layers: model creation refuses it and the shim runs the package's network_predict."""
    cfg = shrink_cfg(rd.path("yolo-voc.cfg"), str(tmp_path / "yolo-voc.cfg"), 96, 96)
    wt = str(tmp_path / "yolo-voc.weights")
    random_weights(cfg, wt, 3)
    same(programs, ["detect", cfg, wt, rd.path("dog.jpg"), rd.path("voc.names"), os.path.join(REF, "darknet"), 0.01, 0.5],
         tmp_path, png=True)
