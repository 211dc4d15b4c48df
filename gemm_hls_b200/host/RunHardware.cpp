// RunHardware.exe N K M [hw|hw_emu] [on|off]
// Drop-in for the reference's device launcher (host/RunHardware.cpp): same argument grammar, same
// stdout sentences (the performance line is what scripts/build_manager.py:601-602 parses), same
// exit codes.  Device work goes through Device.h (Context / Buffer / Kernel over the C-ABI).
//   hw      the H100 selected by $MM_DEVICE (default 0)
//   hw_emu  accepted for compatibility; there is no emulation target, it runs on the H100 as well
//   MM_NUM_GPUS=G (> 1)  C row-blocks over G GPUs inside libmm_b200.so (mm_multi_*): every GPU uploads 1/G of
//                        B, the slices are gathered GPU-to-GPU over NVLink once, no per-step collective
//   MM_POWER_METER=1  NVML power sampling every 10 ms while the kernel is repeated for >= 2 s, then
//                     the reference's "Measured an average power of ... W" line (host/RunHardware.cpp:182-185)
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "Device.h"
#include "HostProblem.h"
#include "PowerMeter.h"

namespace {

struct Options {
  mmhost::Shape shape;
  bool verify = true;
};

int Usage() {
#ifdef MM_DYNAMIC_SIZES
  std::cerr << "Usage: ./RunHardware.exe N K M [<mode [hw/hw_emu]>] [<verify [on/off]>]\n" << std::flush;
#else
  std::cerr << "Usage: ./RunHardware.exe <mode [hw/hw_emu]> [<verify [on/off]>]\n" << std::flush;
#endif
  return 1;
}

// Returns false (after printing the usage) when the command line is malformed.
bool ParseCommandLine(int argc, char **argv, Options *options) {
  const int required = 1 + mmhost::kShapeArguments;
  if (argc < required || argc > required + 2) return false;
  int next = mmhost::ReadShape(argv, 1, &options->shape);
  if (next < argc) {
    const std::string mode(argv[next++]);
    if (mode != "hw" && mode != "hw_emu") return false;
  }
  if (next < argc) {
    const std::string verify(argv[next++]);
    if (verify != "on" && verify != "off") return false;
    options->verify = verify == "on";
  }
  return true;
}

void ReportPerformance(mmhost::Shape const &shape, double device_seconds) {
  const auto gops = 1e-9 * shape.Operations() / device_seconds;
  std::cout << "Kernel executed in " << device_seconds << " seconds, corresponding to a performance of " << gops
            << " GOp/s.\n";
}

int EnvironmentInt(const char *name, int fallback) {
  const char *value = std::getenv(name);
  return value ? std::atoi(value) : fallback;
}

// One GPU: the reference's Context / MakeBuffer / CopyFromHost / MakeKernel / ExecuteTask / CopyToHost
// sequence (host/RunHardware.cpp:116-190).
void RunSingle(mmhost::Problem &problem, bool verify) {
  auto const &shape = problem.shape();
  std::cout << "Initializing CUDA context...\n" << std::flush;
  mm::Context context(EnvironmentInt("MM_DEVICE", 0));

  std::cout << "Initializing device memory...\n" << std::flush;
  auto a_device = context.MakeBuffer<Data_t, mm::Access::read>(shape.CountA());
  auto b_device = context.MakeBuffer<Data_t, mm::Access::read>(shape.CountB());
  auto c_device = context.MakeBuffer<Data_t, mm::Access::write>(shape.CountC());
  if (verify) {
    std::cout << "Copying memory to device...\n" << std::flush;
    a_device.CopyFromHost(problem.A());
    b_device.CopyFromHost(problem.B());
    c_device.CopyFromHost(problem.Result());
  }  // verify off: device buffers stay uninitialised, as in the reference (:99-111)

  std::cout << "Creating kernel...\n" << std::flush;
  auto kernel = context.MakeKernel(kDataTypeCode, kMapOpCode, kReduceOpCode, kKernelFlags, a_device, b_device,
                                   c_device, shape.n, shape.k, shape.m);
  std::cout << "Executing kernel...\n" << std::flush;
  if (EnvironmentInt("MM_POWER_METER", 0) != 0) {
    // A GPU kernel lasts milliseconds and NVML refreshes its reading every ~100 ms: repeat the
    // launch for at least two seconds under the meter and report the last run's time.
    mm::PowerMeter meter(10, static_cast<unsigned>(EnvironmentInt("MM_DEVICE", 0)));  // 10 ms, as the reference
    double device_seconds = 0, total = 0;
    meter.Start();
    do {
      device_seconds = kernel.ExecuteTask().first;
      total += device_seconds;
    } while (total < 2.0);
    meter.Stop();
    ReportPerformance(shape, device_seconds);
    const double watts = meter.AveragePower();
    std::cout << "Measured an average power of " << watts << " W for the GPU ("
              << 1e-9 * shape.Operations() / device_seconds / watts << " GOp/J).\n";
  } else {
    ReportPerformance(shape, kernel.ExecuteTask().first);
  }
  if (verify) {
    std::cout << "Copying back result...\n" << std::flush;
    c_device.CopyToHost(problem.Result());
  }
}

// G GPUs: the same sequence through Device.h's MultiContext (mm_multi_upload / _execute / _download).  The
// reported time is the slowest GPU's kernel time of the SECOND execution: the first one (untimed) loads the
// kernels and sizes the scratch on every device, which the single-GPU ExecuteTask does in its dry run.
void RunMulti(mmhost::Problem &problem, bool verify, int gpus) {
  auto const &shape = problem.shape();
  std::cout << "Initializing " << gpus << " CUDA contexts...\n" << std::flush;
  mm::MultiContext context(gpus);
  std::cout << "Initializing device memory...\n" << std::flush;
  std::vector<Data_t> scratch_a, scratch_b;
  Data_t const *a = problem.A(), *b = problem.B();
  if (!verify) {  // verify off: the reference leaves the buffers uninitialised (:99-111); any bytes will do
    scratch_a.resize(shape.CountA());
    scratch_b.resize(shape.CountB());
    a = scratch_a.data();
    b = scratch_b.data();
  }
  std::cout << "Copying memory to device...\n" << std::flush;
  context.Upload(kDataTypeCode, kKernelFlags, a, b, shape.n, shape.k, shape.m);
  std::cout << "Creating kernel...\n" << std::flush;
  context.Execute(kDataTypeCode, kMapOpCode, kReduceOpCode, kKernelFlags, shape.n, shape.k, shape.m);  // warm-up
  std::cout << "Executing kernel...\n" << std::flush;
  ReportPerformance(shape, context.Execute(kDataTypeCode, kMapOpCode, kReduceOpCode, kKernelFlags, shape.n, shape.k,
                                           shape.m).first);
  if (verify) {
    std::cout << "Copying back result...\n" << std::flush;
    context.Download(kDataTypeCode, problem.Result(), shape.n, shape.m);
  }
}

}  // namespace

int main(int argc, char **argv) {
  Options options;
  if (!ParseCommandLine(argc, argv, &options)) return Usage();
  if (!mmhost::ShapeIsLegal(options.shape, /*verbose=*/true)) return 1;

  mmhost::Problem problem(options.shape);
  std::cout << "Initializing host memory..." << std::flush;
  if (options.verify) {
    problem.DrawInputs();
    problem.AllocateOutputs();
  }
  std::cout << " Done.\n";

  try {
    const int gpus = EnvironmentInt("MM_NUM_GPUS", 1);
    if (gpus > 1) {
      RunMulti(problem, options.verify, gpus);
    } else {
      RunSingle(problem, options.verify);
    }
  } catch (std::runtime_error const &error) {
    std::cerr << "Execution failed with error: \"" << error.what() << "\"." << std::endl;
    return 1;
  }

  if (options.verify) {
    std::cout << "Running reference implementation...\n" << std::flush;
    problem.ComputeExpected();
    std::cout << "Verifying result...\n" << std::flush;
    if (!problem.ResultMatches()) return 1;
    std::cout << "Successfully verified." << std::endl;
  }
  return 0;
}
