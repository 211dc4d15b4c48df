// PrintSpecifications N K M [<SM clock MHz>]
// Counterpart of the reference's specification printer (src/PrintSpecifications.cpp): pure
// arithmetic on the build configuration, no device needed.  For the H100 kernels it reports the
// operation count, the kernel family this configuration dispatches to, that family's pipe-rate
// model, whole-wave runtime estimates, and the reference's communication-volume model
//   Q = N*M*(1 + K/T_N + K/T_M) elements            (src/PrintSpecifications.cpp:72-78)
// evaluated twice: with the CTA tile (bytes through L2) and with the patch of C that the
// co-running tiles share through L2 (bytes from HBM).
#include <algorithm>
#include <cmath>
#include <iomanip>
#include <string>

#include "HostProblem.h"

namespace {

struct KernelModel {
  std::string family;
  double ops_per_sm_clock;  // map+reduce operations per SM per clock of the binding pipe
  unsigned tile_rows, tile_cols, sms_per_tile;
};

KernelModel ModelFor(std::string const &family, mmhost::Shape const &s) {
  // wgmma, dense, per SM and clock: 2048 f16 / 1024 tf32 / 4096 8-bit multiply-adds; 256 x 256 tiles per CTA cluster
  if (family == "wgmma_f16") return {family, 2.0 * 2048, 256, 256, 2};
  if (family == "wgmma_tf32") return {family, 2.0 * 1024, 256, 256, 2};
  if (family == "wgmma_i8") return {family, 2.0 * 4096, 256, 256, 2};
  if (family == "dmma_f64") {
    // DMMA: 128 FMA / clk / SM; 128-row tiles, or 64-row tiles when those fill the last wave better
    // (the launcher's rule, csrc/gemm_dmma.cu: the half-height tile has to win by more than 5 %)
    const double cols = (s.m + 127) / 128;
    const double full = std::ceil(((s.n + 127) / 128) * cols / 132.0), half = 0.5 * 1.05 * std::ceil(((s.n + 63) / 64) * cols / 132.0);
    return {family, 2.0 * 128, half < full ? 64u : 128u, 128, 1};
  }
  // CUDA cores, one warp instruction per scheduler and clock (DESIGN.md 3.3): one Map and one Reduce
  // instruction per element-step, 64 steps / clk / SM
  return {family, 2.0 * 64, 128, 128, 1};
}

template <typename T>
void Row(const char *label, T const &value, const char *unit = "") {
  std::cout << std::left << std::setw(28) << label << value << unit << "\n";
}

}  // namespace

int main(int argc, char **argv) {
  const int required = 1 + mmhost::kShapeArguments;
  if (argc < required || argc > required + 1) {
#ifdef MM_DYNAMIC_SIZES
    std::cerr << "Usage: " << argv[0] << " N K M [<SM clock MHz>]\n" << std::flush;
#else
    std::cerr << "Usage: " << argv[0] << " [<SM clock MHz>]\n" << std::flush;
#endif
    return 1;
  }
  mmhost::Shape s;
  const int next = mmhost::ReadShape(argv, 1, &s);
  const double mhz = next < argc ? std::stod(argv[next]) : 1980.0;  // H100 SXM clocks.max.sm
  constexpr unsigned kSMs = 132;

  const KernelModel model = ModelFor(mm_kernel_path(kDataTypeCode, kMapOpCode, kReduceOpCode, kKernelFlags), s);
  const double ops = 2.0 * s.n * static_cast<double>(s.k) * s.m;
  const double peak_gops = 1e-3 * model.ops_per_sm_clock * kSMs * mhz;
  const unsigned long tiles_n = (s.n + model.tile_rows - 1) / model.tile_rows;
  const unsigned long tiles_m = (s.m + model.tile_cols - 1) / model.tile_cols;
  const unsigned long slots = kSMs / model.sms_per_tile;
  const unsigned long waves = (tiles_n * tiles_m + slots - 1) / slots;
  const double tile_seconds =
      2.0 * model.tile_rows * model.tile_cols * s.k / (model.ops_per_sm_clock * model.sms_per_tile * 1e6 * mhz);
  const double ideal = 1e-9 * ops / peak_gops, expected = static_cast<double>(waves) * tile_seconds;

  Row("Configuration:", std::string(kDataTypeName) + " (" + kMapOpName + ", " + kReduceOpName + ")");
  Row("Kernel family:", model.family);
  Row("Frequency:", mhz, " MHz");
  Row("Number of operations:", ops);
  Row("Ideal performance:", peak_gops, " GOp/s");
  Row("Ideal runtime:", ideal, " seconds");
  Row("Expected runtime:", expected, " seconds (whole waves of full tiles)");
  Row("Percentage of ideal:", 100.0 * ideal / expected, "%");
  Row("Expected performance:", 1e-9 * ops / expected, " GOp/s");
  std::cout << "Compute tiles: " << model.tile_rows << "x" << model.tile_cols << " per "
            << (model.sms_per_tile == 2 ? "CTA pair" : "CTA") << ", " << kSMs << " SMs (" << tiles_n * tiles_m
            << " tiles, " << waves << " waves)\n";
  Row("Tiles in N:", tiles_n);
  Row("Tiles in M:", tiles_m);

  auto volume = [&](double t_n, double t_m) { return static_cast<double>(s.n) * s.m * (1 + s.k / t_n + s.k / t_m); };
  const double through_l2 = volume(model.tile_rows, model.tile_cols);
  // patch shared through L2: 2048 rows (rasterisation group) x the columns the other tiles cover
  const double patch_rows = std::min<double>(2048, s.n);
  const double patch_cols = std::min<double>(s.m, std::max<double>(model.tile_cols, static_cast<double>(slots) * model.tile_rows / patch_rows * model.tile_cols));
  const double from_hbm = volume(patch_rows, patch_cols);
  Row("Communication volume:", through_l2, " elements through L2 (CTA tile)");
  Row("", 1e-9 * through_l2 * sizeof(Data_t), " GB");
  Row("HBM volume model:", from_hbm, " elements (L2 patch as memory tile)");
  Row("", 1e-9 * from_hbm * sizeof(Data_t), " GB");
  Row("I/O access fraction:", through_l2 / (3.0 * s.n * s.m * s.k));
  Row("Algorithmic bytes:", (static_cast<double>(s.n) * s.k + static_cast<double>(s.k) * s.m +
                             static_cast<double>(s.n) * s.m) * sizeof(Data_t));
  return 0;
}
