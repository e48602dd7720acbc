// ORACLE — TEST INFRASTRUCTURE ONLY.  Appended to the generated Eigen stand-in of riganalyzer.mk: the VectorXd name.
#pragma once
namespace Eigen {
typedef Matrix<double, Dynamic, 1> VectorXd;
}  // namespace Eigen
