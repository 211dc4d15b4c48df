// TestSimulation N K M
// Drop-in for the reference's software test (test/TestSimulation.cpp): same arguments, same two
// progress lines, same verdict sentence, same exit codes.  The "simulation" is the real H100 path
// behind the same extern "C" MatrixMultiplicationKernel(a, b, c, n, k, m) call on host pointers.
#include <stdexcept>

#include "HostProblem.h"

namespace {

int Fail(std::runtime_error const &error) {
  std::cerr << "Execution failed with error: \"" << error.what() << "\"." << std::endl;
  return 1;
}

void Launch(mmhost::Problem &problem) {
  auto const &s = problem.shape();
#ifdef MM_DYNAMIC_SIZES
  MatrixMultiplicationKernel(problem.A(), problem.B(), problem.Result(), s.n, s.k, s.m);
#else
  (void)s;
  MatrixMultiplicationKernel(problem.A(), problem.B(), problem.Result());
#endif
}

}  // namespace

int main(int argc, char **argv) {
  if (argc != 1 + mmhost::kShapeArguments) {
    std::cerr << "Usage: ./TestSimulation N K M" << std::endl;
    return 1;
  }
  mmhost::Shape shape;
  mmhost::ReadShape(argv, 1, &shape);
  if (!mmhost::ShapeIsLegal(shape, /*verbose=*/false)) return 1;

  mmhost::Problem problem(shape);
  problem.DrawInputs();
  problem.AllocateOutputs();
  problem.ComputeExpected();

  std::cout << "Running simulation...\n" << std::flush;
  try {
    Launch(problem);
  } catch (std::runtime_error const &error) {
    return Fail(error);
  }

  std::cout << "Verifying results...\n" << std::flush;
  if (!problem.ResultMatches()) return 1;
  std::cout << "Matrix-matrix multiplication successfully verified.\n";
  return 0;
}
