#include <math.h>
#include <stdio.h>
#include <stdint.h>
#include <string.h>
#include <stdlib.h>
#include "../safe_learning_b200/csrc/exp2_tab64.h"
static const double EXP2_TAB[64] = {SLB_EXP2_TAB64};
static inline double exp_neg_tab(double x){
  const double MAGIC = 6755399441055744.0;
  double t = fma(x, 92.332482616893656877, MAGIC);         // 64/ln2
  int64_t bits; memcpy(&bits,&t,8); int n = (int)(int32_t)(bits & 0xffffffff);
  double nd = t - MAGIC;
  double r = fma(nd, -0.01083042469326756, x);       // ln2/64 hi
  r = fma(nd, -2.9815858269852933e-12, r);                 // ln2/64 lo (placeholder, fixed below)
  double p = 1.0/120.0;
  p = fma(p, r, 1.0/24.0);
  p = fma(p, r, 1.0/6.0);
  p = fma(p, r, 0.5);
  p = fma(p, r, 1.0);
  p = p * r;                       // e^r - 1
  double T = EXP2_TAB[n & 63];
  double v = fma(T, p, T);
  int k = n >> 6;
  int64_t vb; memcpy(&vb,&v,8); vb += ((int64_t)k) << 52; memcpy(&v,&vb,8);
  return x < -700.0 ? 0.0 : v;
}
int main(){
  double maxulp=0; int nbad=0; srand(1);
  for(long i=0;i<20000000;i++){
    double u = rand()/(double)RAND_MAX, w=rand()/(double)RAND_MAX;
    double x = -(u*u*u)*50.0 - w*1e-3;
    if(i%7==0) x = -u*700.0;
    double a=exp_neg_tab(x), b=exp(x);
    double ulp = fabs(a-b)/(nextafter(b,INFINITY)-b);
    if(ulp>maxulp) maxulp=ulp; if(ulp>1.0) nbad++;
  }
  printf("max ulp err %.3f, >1ulp: %d\n",maxulp,nbad);
  return 0;
}
