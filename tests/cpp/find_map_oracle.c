/* Plain-C restatement of find_map_haplotypes (core/tools/read_assigner.cpp:45-64) with maths::almost_equal (utils/maths.hpp:68-71),
 * the checker of phmm_assign_reads' top sets. Built by tests/find_map_oracle.py with -ffp-contract=off: every operation is rounded on
 * its own, as the reference's expression is written. */
#include <float.h>
#include <math.h>
#include <stdint.h>

static int almost_equal(const double lhs, const double rhs)
{
    const int ulp = 1;
    return lhs == rhs || fabs(lhs - rhs) < DBL_EPSILON * fabs(lhs + rhs) * ulp;
}

/* One read against the n <= 64 haplotypes of its genotype: likelihoods[k] + log_priors[k] (log_priors NULL = zeros, get_priors :36-43).
 * Returns the set as a mask, bit k = haplotype k. */
uint64_t oracle_find_map_haplotypes(const int n, const double* likelihoods, const double* log_priors)
{
    uint64_t result = 0;
    double max_likelihood = -DBL_MAX;                    /* std::numeric_limits<double>::lowest() */
    for (int k = 0; k < n; ++k) {
        const double curr = likelihoods[k] + (log_priors ? log_priors[k] : 0.0);
        if (almost_equal(curr, max_likelihood)) {
            result |= (uint64_t)1 << k;
        } else if (curr > max_likelihood) {
            result = (uint64_t)1 << k;
            max_likelihood = curr;
        }
    }
    if (result == 0) result = n == 64 ? ~(uint64_t)0 : (((uint64_t)1 << n) - 1);
    return result;
}

/* Every read of a group: lnl is the group's [n][R] matrix (haplotype-major, as phmm_assign_reads returns it). */
void oracle_find_map_group(const int n, const int R, const double* lnl, const double* log_priors, uint64_t* top)
{
    double column[64];
    for (int r = 0; r < R; ++r) {
        for (int k = 0; k < n; ++k) column[k] = lnl[(long long)k * R + r];
        top[r] = oracle_find_map_haplotypes(n, column, log_priors);
    }
}
