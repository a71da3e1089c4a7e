// TEST INFRASTRUCTURE ONLY: the EMU_DCAL flag of the query harnesses (include after the kernel file).
//   EMU_DCAL=1       the launch reads its camera from "device" memory -- a single-map MpBatch whose calibs point at one
//                    12-float buffer holding in.bin's calib -- while MpCalib::m holds NaNs, so any read of the by-value camera
//                    shows in the output.
//   EMU_DCAL=<file>  two launches read that one buffer: the first with the file's 12 float32 (its output goes to <out>.first),
//                    the second, after the buffer has been rewritten, with in.bin's (to <out>).
#pragma once
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>

// run(const MpBatch* bt, const char* out_path) -> exit code: one launch (bt == nullptr: the by-value camera) and its output
template <class Run>
static int emu_dcal_run(MpCalib& cal, const float* calib, const char* out_path, Run run) {
  const char* flag = getenv("EMU_DCAL");
  if (!flag) return run(static_cast<const MpBatch*>(nullptr), out_path);
  static float buf[12];
  MpBatch bt;
  bt.calibs = buf;
  for (int k = 0; k < 12; ++k) cal.m[k] = NAN;
  if (strcmp(flag, "1") != 0) {
    FILE* f = fopen(flag, "rb");
    const bool ok = f && fread(buf, 4, 12, f) == 12;
    if (f) fclose(f);
    if (!ok) { fprintf(stderr, "EMU_DCAL: cannot read 12 floats from %s\n", flag); return 2; }
    const int rc = run(static_cast<const MpBatch*>(&bt), (std::string(out_path) + ".first").c_str());
    if (rc) return rc;
  }
  memcpy(buf, calib, sizeof(buf));
  return run(static_cast<const MpBatch*>(&bt), out_path);
}
